#!/usr/bin/env python
"""Write-only / read-only / copy bandwidth of this GPU (context for the HBM-bound kernels'
roofline fractions: MEASURED_PEAKS.json holds the copy figure only).  Run on an H100."""
import json

import torch


def timeit(fn, n=10):
    fn()
    torch.cuda.synchronize()
    best = 1e9
    for _ in range(n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1))
    return best


def main():
    n = 1 << 29   # 2 GiB of fp32
    a = torch.empty(n, device='cuda')
    b = torch.empty(n, device='cuda')
    a.normal_()
    out = {}
    out['write_only_gbs'] = round(n * 4 / timeit(lambda: b.zero_()) / 1e6, 1)
    out['fill_gbs'] = round(n * 4 / timeit(lambda: b.fill_(1.5)) / 1e6, 1)
    out['read_only_gbs'] = round(n * 4 / timeit(lambda: a.sum()) / 1e6, 1)
    out['copy_gbs_read_plus_write'] = round(2 * n * 4 / timeit(lambda: b.copy_(a)) / 1e6, 1)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
