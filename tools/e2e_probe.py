"""Where does the end-to-end (host buffers in / out) step spend its time?

Runs the DfM.simple_test hot-path segment (HotPathPipeline) on an H100 in four ways and prints
one JSON line: (a) per-kernel profile of one synchronous frame, (b) asynchronous loop with all
copies (what bench.py reports as e2e), (c) the same loop fed the SAME already-staged pair (no
H2D of the pair), (d) the same without collecting outputs on the host path differences.
"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    import torch

    import bench
    from depth_from_motion_b200 import capi, modules
    from depth_from_motion_b200 import synthetic as syn

    H, W, D, C = bench.H, bench.W, bench.D, bench.C
    capi.lib()
    pairs = []
    for i in range(2):
        cur, prev, metas, params = syn.make_kitti_pair(100 + i, H, W, D, ori_shape=bench.ORI_SHAPE)
        metas[0]['cam2img'] = syn.KITTI_P2.astype('float32').tolist()
        pairs.append((metas, cur.pin_memory(), prev.pin_memory()))
    cfg = syn.depth_cfg_for(D)
    model = modules.DfMBackbone(in_channels=C, depth_cfg=cfg).cuda().eval()
    model.load_state_dict(params, strict=True)
    model.downsampled_depth = bench._depths(cfg, 4)
    head = modules.DepthHead(
        depth_cfg=dict(mode='UD', num_bins=cfg['num_bins'], min_depth=2, max_depth=59.6),
        with_convs=False, num_views=1, depth_loss=dict(type='ce', loss_weight=1.0))
    head.depth_samples = bench._depths(cfg, 1)
    head.downsample_factor = 4
    fc = syn.make_frustum_case(7, H, W, D, (288, 304, 20))
    frustum = modules.FrustumToVoxel().eval()
    frustum.load_state_dict(fc['params'], strict=True)
    frustum = frustum.cuda()
    frustum.coordinates_3d = fc['coordinates_3d']
    frustum.depth_cfg = cfg
    h_sem = fc['sem'].contiguous().pin_memory()
    pipe = modules.HotPathPipeline(model, head, frustum)

    cur_d0, prev_d0 = pairs[0][1].cuda(), pairs[0][2].cuda()

    def sync_step(i):
        metas, hc, hp = pairs[i % 2]
        return pipe(hc, hp, h_sem, metas)

    for i in range(3):
        sync_step(i)
    out = {}
    # (a) per-kernel profile of synchronous frames
    capi.profile_enable(True)
    capi.profile_report()
    n = 4
    for i in range(n):
        sync_step(i)
    prof = capi.profile_report()
    capi.profile_enable(False)
    out['profile_ms_per_frame'] = {k: round(v['ms'] / n, 4)
                                   for k, v in sorted(prof.items(), key=lambda kv: -kv[1]['ms'])}
    out['profile_sum_ms'] = round(sum(v['ms'] for k, v in prof.items()
                                      if not k.endswith('_total')) / n, 3)

    def loop(steps, prefetch, same_pair):
        def submit(i):
            metas, hc, hp = pairs[0 if same_pair else i % 2]
            if prefetch:
                nxt = pairs[0 if same_pair else (i + 1) % 2]
                pipe.prefetch(nxt[1], nxt[2], h_sem)
            pipe.submit(hc, hp, h_sem, metas)
        if prefetch:
            pipe.prefetch(pairs[0][1], pairs[0][2], h_sem)
        submit(0)
        submit(1)
        pipe.wait()
        pipe.wait()
        if prefetch:
            pipe.prefetch(pairs[0][1], pairs[0][2], h_sem)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        submit(0)
        host_submit = 0.0
        for i in range(1, steps):
            ts = time.perf_counter()
            submit(i)
            host_submit += time.perf_counter() - ts
            pipe.wait()
        pipe.wait()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / steps, host_submit * 1e3 / (steps - 1)

    steps = 20
    out['async_prefetch_ms'], out['host_submit_ms'] = loop(steps, True, False)

    # per-frame device spans on the compute stream: [a_i, b_i] brackets frame i's enqueued work
    def spans(prefetch):
        ea = [torch.cuda.Event(enable_timing=True) for _ in range(steps)]
        eb = [torch.cuda.Event(enable_timing=True) for _ in range(steps)]

        def submit(i):
            metas, hc, hp = pairs[i % 2]
            if prefetch:
                nxt = pairs[(i + 1) % 2]
                pipe.prefetch(nxt[1], nxt[2], h_sem)
            ea[i].record()
            pipe.submit(hc, hp, h_sem, metas)
            eb[i].record()
        if prefetch:
            pipe.prefetch(pairs[0][1], pairs[0][2], h_sem)
        torch.cuda.synchronize()
        submit(0)
        for i in range(1, steps):
            submit(i)
            pipe.wait()
        pipe.wait()
        torch.cuda.synchronize()
        busy = [ea[i].elapsed_time(eb[i]) for i in range(steps)]
        gap = [eb[i].elapsed_time(ea[i + 1]) for i in range(steps - 1)]
        return dict(frame_span_ms=round(sum(busy[2:]) / len(busy[2:]), 3),
                    gap_ms=round(sum(gap[2:]) / len(gap[2:]), 3),
                    spans=[round(b, 2) for b in busy[:8]], gaps=[round(g, 2) for g in gap[:8]])
    # per-kernel profile while the asynchronous loop runs, against the synchronous one
    capi.profile_enable(True)
    capi.profile_report()
    loop(steps, True, False)
    prof_a = capi.profile_report()
    capi.profile_enable(False)
    na = steps + 2
    out['async_profile_sum_ms'] = round(sum(v['ms'] for k, v in prof_a.items()
                                            if not k.endswith('_total')) / na, 3)
    out['async_vs_sync_kernel_ms'] = {
        k: [round(v['ms'] / na, 4), out['profile_ms_per_frame'].get(k)]
        for k, v in sorted(prof_a.items(), key=lambda kv: -kv[1]['ms'])}

    # clocks / power while a long asynchronous loop runs
    try:
        import threading
        import pynvml
        pynvml.nvmlInit()
        hnd = pynvml.nvmlDeviceGetHandleByIndex(0)
        samples, stop = [], [False]

        def sampler():
            while not stop[0]:
                samples.append((pynvml.nvmlDeviceGetClockInfo(hnd, pynvml.NVML_CLOCK_SM),
                                pynvml.nvmlDeviceGetPowerUsage(hnd) / 1000.0,
                                pynvml.nvmlDeviceGetCurrentClocksThrottleReasons(hnd)))
                time.sleep(0.02)
        th = threading.Thread(target=sampler)
        th.start()
        ms_long, _ = loop(100, True, False)
        stop[0] = True
        th.join()
        out['long_async_ms'] = ms_long
        out['nvml'] = dict(sm_mhz=[s_[0] for s_ in samples][::4], power_w=[round(s_[1]) for s_ in samples][::4],
                           reasons=sorted({hex(s_[2]) for s_ in samples}))
        samples.clear()
        stop[0] = False
        th = threading.Thread(target=sampler)
        th.start()
        t0 = time.perf_counter()
        for _ in range(100):
            model(cur_d0, prev_d0, pairs[0][0])
        torch.cuda.synchronize()
        out['long_device_backbone_ms'] = (time.perf_counter() - t0) * 1e3 / 100
        stop[0] = True
        th.join()
        out['nvml_device_loop'] = dict(sm_mhz=[s_[0] for s_ in samples][::4],
                                       power_w=[round(s_[1]) for s_ in samples][::4],
                                       reasons=sorted({hex(s_[2]) for s_ in samples}))
    except Exception as exc:  # noqa
        out['nvml_error'] = repr(exc)
    out['spans_prefetch'] = spans(True)
    out['spans_noprefetch'] = spans(False)

    # compute only: device-resident inputs through the module API (backbone -> depth head
    # reduction + FrustumToVoxel is inside pipeline only, so time backbone alone and the
    # pipeline's frustum share separately via the profile above)
    cur_d, prev_d = pairs[0][1].cuda(), pairs[0][2].cuda()
    for _ in range(3):
        model(cur_d, prev_d, pairs[0][0])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        model(cur_d, prev_d, pairs[0][0])
    torch.cuda.synchronize()
    out['backbone_device_loop_ms'] = (time.perf_counter() - t0) * 1e3 / steps

    # raw PCIe rates for the buffers used here
    big = pairs[0][1]
    dev = torch.empty_like(big, device='cuda')
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(10):
        dev.copy_(big, non_blocking=True)
    torch.cuda.synchronize()
    out['h2d_gbs'] = big.numel() * 4 * 10 / (time.perf_counter() - t0) / 1e9
    hv = pipe._outs[0][0]
    dv = torch.empty_like(hv, device='cuda')
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(10):
        hv.copy_(dv, non_blocking=True)
    torch.cuda.synchronize()
    out['d2h_gbs'] = hv.numel() * 4 * 10 / (time.perf_counter() - t0) / 1e9
    out['async_noprefetch_ms'], _ = loop(steps, False, False)
    # sync loop (no overlap at all)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        sync_step(i)
    torch.cuda.synchronize()
    out['sync_ms'] = (time.perf_counter() - t0) * 1e3 / steps
    print(json.dumps(out))


if __name__ == '__main__':
    main()
