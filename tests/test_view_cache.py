"""The detectors' per-view image-feature cache (``DfM.set_feature_cache``).

CPU: a numpy restatement of ``dfm_view_fingerprint`` and its sensitivity; the cache policy
(LRU, capacity, deduplication, forced views, invalidation, counters) with a fake fingerprint
and a fake feature function.

GPU: the fingerprint and ``dfm_views_equal`` kernels bit for bit; lifting through a pointer
table against the contiguous entry point; KITTI and Waymo 10-sweep video sequences whose every
call equals the same call with the cache off, with the expected hit counts; forced fingerprint
collisions; weight changes between calls; and the cache-off path launching no cache kernel.
"""
import copy
import ctypes
import hashlib

import numpy as np
import pytest
import torch

from depth_from_motion_b200 import capi, checkpoint, image_prep, modules
from depth_from_motion_b200 import synthetic as syn

from .test_detector import KITTI, SWEEPS10, _free, _same, build, random_state

K0, K1 = 0x9E3779B97F4A7C15, 0xC2B2AE3D27D4EB4F
M1, M2 = 0xBF58476D1CE4E5B9, 0x94D049BB133111EB


def _mix(words, key, mul):
    """The per-word contribution of view_cache_kernels.cuh (uint64 arithmetic wraps)."""
    i = np.arange(words.size, dtype=np.uint64)
    x = ((words.astype(np.uint64) << np.uint64(32)) ^ i ^ np.uint64(key)) * np.uint64(mul)
    return x ^ (x >> np.uint64(32))


def np_fingerprint(view):
    """128-bit fingerprint of one fp32 view: two lanes, each the sum mod 2^64 of the mixed
    (bits, index) words."""
    words = np.ascontiguousarray(view, dtype=np.float32).reshape(-1).view(np.uint32)
    return tuple(int(_mix(words, k, m).sum(dtype=np.uint64)) for k, m in ((K0, M1), (K1, M2)))


# ---------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------
def test_fingerprint_restatement_sees_every_bit_swaps_and_signed_zero():
    rng = np.random.RandomState(0)
    v = rng.standard_normal(1003).astype(np.float32)
    base = np_fingerprint(v)
    words = v.view(np.uint32)
    for pos in (0, 1, 500, 1002):
        for bit in (0, 7, 22, 23, 31):
            w = words.copy()
            w[pos] ^= np.uint32(1 << bit)
            assert np_fingerprint(w.view(np.float32)) != base, (pos, bit)
    for i, j in ((0, 1), (3, 999), (0, 1002)):
        s = v.copy()
        s[i], s[j] = s[j], s[i]
        assert np_fingerprint(s) != base, (i, j)
    z = np.zeros(8, np.float32)
    nz = z.copy()
    nz[5] = -0.0
    assert np_fingerprint(z) != np_fingerprint(nz)
    # summation order: the lanes are sums of per-word terms, so any order gives the same bits
    for k, m in ((K0, M1), (K1, M2)):
        terms = _mix(words, k, m)
        perm = rng.permutation(terms.size)
        assert int(terms[perm].sum(dtype=np.uint64)) == int(terms.sum(dtype=np.uint64))
        halves = np.array([terms[perm[:400]].sum(dtype=np.uint64),
                           terms[perm[400:]].sum(dtype=np.uint64)])
        assert int(halves.sum(dtype=np.uint64)) == int(terms.sum(dtype=np.uint64))


def _fake_fingerprints(batch):
    out = []
    for v in batch:
        d = hashlib.sha256(v.contiguous().numpy().tobytes()).digest()
        out.append((int.from_bytes(d[:8], 'little'), int.from_bytes(d[8:16], 'little')))
    return out


def _fake_equal(pairs):
    return [torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in pairs]


@pytest.fixture
def fakes(monkeypatch):
    calls = dict(fingerprint=0)

    def fp(batch):
        calls['fingerprint'] += 1
        return _fake_fingerprints(batch)
    monkeypatch.setattr(modules, '_view_fingerprints', fp)
    monkeypatch.setattr(modules, '_views_equal', _fake_equal)
    return calls


class Features:
    """Fake feature function: feature = view * 2, records the views it is given."""

    def __init__(self):
        self.seen = []

    def __call__(self, views):
        self.seen.append(len(views))
        return [(v * 2, 'extra') for v in views]


def _view(seed):
    return torch.from_numpy(np.random.RandomState(seed).standard_normal((3, 4, 5))
                            .astype(np.float32))


def test_cache_lru_order_and_capacity(fakes):
    c = modules._ViewFeatureCache(2)
    f = Features()
    A, B, C = _view(1), _view(2), _view(3)
    state = lambda check: 's'  # noqa: E731
    for v in (A, B):
        c.run(v[None], f, state)
    r = c.run(A[None], f, state)                      # hit, refreshes A
    assert torch.equal(r[0][0], A * 2) and r[0][1] is None
    c.run(C[None], f, state)                          # evicts B, the least recently used
    assert c.stats()['views'] == 2
    c.run(A[None], f, state)                          # still there
    assert c.stats()['hits'] == 2
    c.run(B[None], f, state)                          # was evicted
    assert c.stats() == dict(hits=2, misses=4, rejected=0, views=2,
                             bytes=2 * 2 * A.numel() * 4)
    assert f.seen == [1, 1, 1, 1]


def test_cache_deduplicates_within_a_call_and_computes_forced_views(fakes):
    c = modules._ViewFeatureCache(8)
    f = Features()
    A, B = _view(1), _view(2)
    state = lambda check: 0  # noqa: E731
    r = c.run(torch.stack([A, B, A.clone(), B.clone()]), f, state)
    assert f.seen == [2]
    assert [x[1] for x in r] == ['extra', 'extra', None, None]
    assert all(torch.equal(x[0], v * 2) for x, v in zip(r, (A, B, A, B)))
    assert c.stats()['misses'] == 2 and c.stats()['hits'] == 2 and c.stats()['views'] == 2
    # a forced view is computed even when cached; the other one is served
    r = c.run(torch.stack([A, B]), f, state, forced=(0,))
    assert f.seen == [2, 1] and r[0][1] == 'extra' and r[1][1] is None
    # a state change drops the entries recorded under the old one
    c.run(torch.stack([A, B]), f, lambda check: 1)
    assert f.seen == [2, 1, 2]


def test_cache_rejects_fingerprint_collisions(monkeypatch):
    monkeypatch.setattr(modules, '_view_fingerprints', lambda batch: [(7, 7)] * len(batch))
    monkeypatch.setattr(modules, '_views_equal', _fake_equal)
    c = modules._ViewFeatureCache(8)
    f = Features()
    A, B = _view(1), _view(2)
    r = c.run(torch.stack([A, B]), f, lambda check: 0)
    assert torch.equal(r[1][0], B * 2) and c.stats()['rejected'] == 1
    r = c.run(B[None], f, lambda check: 0)
    assert torch.equal(r[0][0], B * 2) and c.stats()['rejected'] == 2
    r = c.run(B[None], f, lambda check: 0)            # B replaced A under the shared key
    assert c.stats()['hits'] == 1 and c.stats()['rejected'] == 2


def _cpu_kitti_with_cache(max_views):
    """DfM on the CPU with the image modules' parameter sync primed as a forward leaves it."""
    det = build(KITTI).eval()
    det.set_feature_cache(max_views)
    noop = lambda *a: None  # noqa: E731
    for m in (det.backbone, det.neck):
        m._sync = modules._ParamSync()
        m._sync.sync(m, noop)

    def compute(views):
        for m in (det.backbone, det.neck):            # what the real forwards do first
            m._sync.sync(m, noop)
        return [(v + 1, None) for v in views]
    A = _view(5)

    def call():
        before = det.feature_cache_stats()['hits']
        det._feature_cache.run(A[None], compute,
                               lambda check: det._feature_cache_state('cpu', check))
        return det.feature_cache_stats()['hits'] > before
    return det, call


def test_cache_empties_on_weight_uploads_train_and_conv_impl(fakes):
    det, call = _cpu_kitti_with_cache(4)
    assert not call() and call()
    det.load_state_dict(det.state_dict())
    assert not call() and call()
    det.backbone.sync_params()
    assert not call() and call()
    det.neck.sync_params()
    assert not call() and call()
    with torch.no_grad():
        det.backbone.conv1.weight.add_(0)             # in place through the parameter
    assert not call() and call()
    det.train()
    det.eval()
    assert det.feature_cache_stats()['views'] == 0
    assert not call() and call()
    det.neck.conv_impl = 'simt'
    assert not call() and call()
    # a new generation (an upload the cache did not see coming) also drops the entries
    det.backbone._sync.generation += 1
    assert not call() and call()
    stats = det.feature_cache_stats()
    assert stats['hits'] == 8 and stats['misses'] == 8 and stats['rejected'] == 0
    det.set_feature_cache(4)
    assert det.feature_cache_stats() == dict(hits=0, misses=0, rejected=0, views=0, bytes=0)


def test_cache_off_never_fingerprints(fakes):
    class Call(torch.nn.Module):
        def __init__(self, fn):
            super().__init__()
            self.fn = fn

        def forward(self, *args):
            return self.fn(*args)
    det = build(KITTI).eval()
    det.set_feature_cache(0)
    det.backbone = Call(lambda x: (x[:, :1],))
    det.neck = Call(lambda feats: (feats[0], feats[0]))
    det.backbone_stereo = Call(lambda c, p, metas: (c,) * 3)
    det.extract_feat(torch.zeros(1, 2, 3, 8, 8), [dict(cur2prevs=syn.KITTI_CUR2PREV[2:3])])
    assert fakes['fingerprint'] == 0
    with pytest.raises(ValueError):
        det.set_feature_cache(-1)


# ---------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------
def _gpu_fingerprints(batch):
    return modules._view_fingerprints(batch)


@pytest.mark.gpu
@pytest.mark.parametrize('n,elems,offset', [(1, 1, 0), (1, 7, 0), (3, 1001, 1), (4, 4096, 2),
                                            (2, 3 * 832 * 1248, 0), (10, 3 * 832 * 1248, 0)])
def test_fingerprint_kernel_equals_the_restatement(n, elems, offset):
    g = torch.Generator().manual_seed(n * 7 + elems)
    buf = torch.randn(n * elems + offset, generator=g)
    host = buf[offset:].reshape(n, elems)
    dev = buf.cuda()[offset:].reshape(n, elems)       # offset: a view not 16-byte aligned
    got = _gpu_fingerprints(dev)
    again = _gpu_fingerprints(dev)
    capi.sync_check()
    assert got == again
    step = max(1, n // 3) if elems > 10 ** 6 else 1    # the numpy restatement is slow at 3M
    for v in range(0, n, step):
        assert got[v] == np_fingerprint(host[v].numpy()), v
    assert len(set(got)) == n


@pytest.mark.gpu
def test_views_equal_kernel():
    g = torch.Generator().manual_seed(3)
    a = torch.randn(5, 4099, generator=g)
    b = a.clone()
    b[1, 0] = float(np.nextafter(np.float32(b[1, 0]), np.float32(np.inf)))
    b[2, -1] = float(np.nextafter(np.float32(b[2, -1]), np.float32(-np.inf)))
    a[3].zero_()
    b[3].zero_()
    b.view(torch.int32)[3, 17] = -0x80000000          # -0.0
    a.view(torch.int32)[4, 9] = 0x7FC00000            # two quiet-NaN payloads
    b.view(torch.int32)[4, 9] = 0x7FC00001
    da, db = a.cuda(), b.cuda()
    got = modules._views_equal([(da[i], db[i]) for i in range(5)])
    assert got == [True, False, False, False, False]
    # 16-byte aligned rows of a multiple of 4 words take the vector path
    x = torch.randn(70, 4096, generator=g).cuda()
    y = x.clone()
    y[65, 4095] += 1
    got = modules._views_equal([(x[i], y[i]) for i in range(70)])
    assert got == [i != 65 for i in range(70)]
    capi.sync_check()


def _lift_case():
    rng = np.random.RandomState(41)
    t, nv, c, hf, wf = 2, 3, 64, 20, 32
    feats = torch.from_numpy(rng.standard_normal((t * nv, c, hf, wf)).astype(np.float32))
    mats = []
    for f in range(t):
        for v in range(nv):
            yaw = (v - 1) * 0.6
            r = np.array([[np.cos(yaw), np.sin(yaw), 0], [-np.sin(yaw), np.cos(yaw), 0],
                          [0, 0, 1]])
            ext = np.eye(4)
            ext[:3, :3] = np.array([[0, -1, 0], [0, 0, -1], [1, 0, 0]], dtype=np.float64) @ r
            ext[:3, 3] = ext[:3, :3] @ np.array([-0.5 * f, 0.1 * v, 0.3])
            k = np.array([[60., 0, 64, 0], [0, 60., 40, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
            mats.append(k @ ext)
    meta = dict(ori_lidar2img=np.array(mats), input_shape=(80, 128),
                img_shape=[(78, 125, 3)] * (t * nv), scale_factor=1.0)
    return feats, meta, [12, 10, 4], [2.0, -10.0, -2.0, 26.0, 10.0, 2.0], t, nv


@pytest.mark.gpu
@pytest.mark.parametrize('agg', ['mean', 'concat'])
@pytest.mark.parametrize('channels_last', [True, False])
def test_lift_through_a_pointer_table_equals_the_contiguous_entry(monkeypatch, agg,
                                                                  channels_last):
    feats, meta, nvox, vrange, t, nv = _lift_case()
    dev = feats.cuda()
    # separate allocations in shuffled order, with gaps between them
    order = np.random.RandomState(2).permutation(t * nv)
    keep, views = [], [None] * (t * nv)
    for s in order:
        keep.append(torch.empty(4099, device='cuda'))
        views[s] = dev[s].clone()
    got = modules.multiview_lift(views, meta, nvox, vrange, nv, t, agg,
                                 channels_last=channels_last)
    L = capi.lib()
    name = 'dfm_multiview_lift_views_cl' if channels_last else 'dfm_multiview_lift_views'
    contiguous = getattr(L, name.replace('_views', ''))
    # the same call routed to the contiguous entry (table[0] is the start of `dev`)
    monkeypatch.setattr(L, name, lambda desc, table, *rest: contiguous(
        desc, ctypes.c_void_p(table[0]), *rest))
    ref = modules.multiview_lift(dev, meta, nvox, vrange, nv, t, agg,
                                 channels_last=channels_last)
    capi.sync_check()
    assert torch.equal(got, ref)
    assert float(ref.abs().sum()) > 0


def _gpu_detector(name, seed=11):
    _free()
    det = build(name)
    checkpoint.load_detector(random_state(det, seed), det)
    return det.cuda().eval()


def _kitti_frames(n):
    rng = np.random.RandomState(12)
    base = (127 + 100 * np.tanh(syn.smooth_field(rng, 3, 375, 1242 + 4 * n, cell=16)[0].numpy()))
    base = base.astype(np.uint8).transpose(1, 2, 0)
    return [np.ascontiguousarray(base[:, 4 * (n - i):4 * (n - i) + 1242]) for i in range(n)]


def _kitti_call(frames, t):
    return image_prep.prepare_kitti(frames[t], [frames[t - 1]], syn.KITTI_P2,
                                    syn.KITTI_CUR2PREV[2:3])


def _run(det, inputs):
    with torch.no_grad():
        return det.simple_test(inputs[0], copy.deepcopy(inputs[1]))


@pytest.mark.gpu
def test_kitti_sequence_equals_cache_off():
    det = _gpu_detector(KITTI)
    try:
        frames = _kitti_frames(5)
        calls = [_kitti_call(frames, t) for t in range(1, 5)]
        off = [_run(det, c) for c in calls]
        launches_off = []
        for c in calls[:2]:
            n0 = capi.launch_counters()[0]
            _run(det, c)
            launches_off.append(capi.launch_counters()[0] - n0)
        sizes = []
        hook = det.backbone.register_forward_pre_hook(lambda m, a: sizes.append(a[0].shape[0]))
        det.set_feature_cache(4)
        for k, c in enumerate(calls):
            _same(_run(det, c), off[k], f'kitti call {k}')
            st = det.feature_cache_stats()
            assert (st['hits'], st['misses'], st['rejected']) == (k, k + 2, 0), st
        hook.remove()
        assert sizes == [2, 1, 1, 1]
        assert det.feature_cache_stats()['views'] == 4
        capi.sync_check()
        # the cache off again: the launches of a call are what they were before it was on, and
        # no cache kernel runs
        det.set_feature_cache(0)
        capi.profile_enable(True)
        capi.profile_report()
        n0 = capi.launch_counters()[0]
        _same(_run(det, calls[0]), off[0], 'kitti off again')
        assert capi.launch_counters()[0] - n0 == launches_off[0] == launches_off[1]
        torch.cuda.synchronize()
        prof = capi.profile_report()
        capi.profile_enable(False)
        assert not any(k.startswith('view') for k in prof), sorted(prof)
    finally:
        capi.profile_enable(False)
        _free(det)


@pytest.mark.gpu
def test_kitti_forced_collisions_are_rejected(monkeypatch):
    det = _gpu_detector(KITTI)
    try:
        frames = _kitti_frames(4)
        calls = [_kitti_call(frames, t) for t in range(1, 4)]
        off = [_run(det, c) for c in calls]
        monkeypatch.setattr(modules, '_view_fingerprints', lambda batch: [(1, 2)] * len(batch))
        det.set_feature_cache(4)
        for k, c in enumerate(calls):
            _same(_run(det, c), off[k], f'collision call {k}')
        st = det.feature_cache_stats()
        # every call: prev shares cur's key and differs from it
        assert (st['hits'], st['misses'], st['rejected']) == (0, 6, 3), st
    finally:
        _free(det)


@pytest.mark.gpu
def test_kitti_weight_changes_between_calls():
    det = _gpu_detector(KITTI)
    try:
        frames = _kitti_frames(4)
        a, b, c = [_kitti_call(frames, t) for t in range(1, 4)]
        det.set_feature_cache(4)
        _run(det, a)
        _run(det, b)                                   # prev (frame 1) from the cache
        state = det.state_dict()
        state['backbone.layer1.0.conv1.weight'] = state['backbone.layer1.0.conv1.weight'] * 1.5
        det.load_state_dict(state)
        got = _run(det, b)
        assert det.feature_cache_stats()['hits'] == 1  # nothing served after the load
        det.set_feature_cache(0)
        _same(got, _run(det, b), 'after load_state_dict')
        det.set_feature_cache(4)
        _run(det, c)
        _run(det, c)
        assert det.feature_cache_stats()['hits'] == 1
        det.backbone.layer1[0].conv2.weight.data[0, 0, 1, 1] += 0.25
        det.backbone.sync_params()
        got = _run(det, c)
        assert det.feature_cache_stats()['hits'] == 1  # nothing served after sync_params
        det.set_feature_cache(0)
        _same(got, _run(det, c), 'after sync_params')
        capi.sync_check()
    finally:
        _free(det)


def _waymo_frames(n):
    g = torch.Generator(device='cuda').manual_seed(5)
    return [[torch.randint(0, 256, (1280, 1920, 3), dtype=torch.uint8, device='cuda',
                           generator=g) for _ in range(5)] for _ in range(n)]


@pytest.mark.gpu
def test_waymo_10sweep_sequence_equals_cache_off():
    det = _gpu_detector(SWEEPS10, 21)
    try:
        frames = _waymo_frames(12)
        ori = np.diag([1 / 0.65, 1 / 0.65, 1, 1]) @ syn.waymo_lidar2img(2)

        def call(t):    # the reference frame ten back; frame 0 stands in at the start
            views = frames[t] + frames[max(t - 10, 0)]
            return image_prep.prepare_waymo(views, ori, num_ref_frames=1)
        off = [_run(det, call(t)) for t in range(12)]
        # LRU with refresh: the last 10 current frames plus the 10 references they hit
        det.set_feature_cache(100)
        for t in range(12):
            _same(_run(det, call(t)), off[t], f'waymo t={t}')
            st = det.feature_cache_stats()
            # call 0: five views computed, their copies as references served; then the
            # current views are computed and the reference frame is served
            assert (st['hits'], st['misses'], st['rejected']) == (5 * (t + 1), 5 * (t + 1), 0)
        assert det.feature_cache_stats()['views'] == 60
        # room for one frame only: a call that computes both of its frames keeps the one it
        # stored last, the reference frame 0, which the next call hits; no later reference
        # frame is ever served.  The results stay equal throughout.
        det.set_feature_cache(5)
        for t in range(12):
            _same(_run(det, call(t)), off[t], f'waymo small t={t}')
        st = det.feature_cache_stats()
        assert (st['hits'], st['misses'], st['views']) == (30, 90, 5), st
        capi.sync_check()
    finally:
        _free(det)


@pytest.mark.gpu
def test_waymo_10sweep_recovers_from_a_fresh_reference_frame():
    """One call whose reference frame no call has seen computes 10 views instead of 5: the
    image modules keep their handles across that batch change, so the entries stored before it
    stay valid and the next call is served again."""
    det = _gpu_detector(SWEEPS10, 21)
    try:
        frames = _waymo_frames(25)
        fresh = frames.pop()
        ori = np.diag([1 / 0.65, 1 / 0.65, 1, 1]) @ syn.waymo_lidar2img(2)

        def call(t):
            ref = fresh if t == 11 else frames[max(t - 10, 0)]
            return image_prep.prepare_waymo(frames[t] + ref, ori, num_ref_frames=1)
        off = [_run(det, call(t)) for t in range(24)]
        det.set_feature_cache(100)
        hits, handles = [], None
        for t in range(24):
            before = det.feature_cache_stats()['hits']
            _same(_run(det, call(t)), off[t], f'waymo fresh t={t}')
            hits.append(det.feature_cache_stats()['hits'] - before)
            now = [(m._handle.value, m._sync) for m in (det.backbone, det.neck)]
            assert handles is None or now == handles, f'handle re-created at t={t}'
            handles = now
        assert hits == [5] * 11 + [0] + [5] * 12, hits
        assert det.feature_cache_stats()['rejected'] == 0
        capi.sync_check()
    finally:
        _free(det)
