"""Times the stand-alone fp32 kernels of the layer-primitive API with CUDA events: the four resize modes forward and backward
(cis_resize_f32 / cis_resize_f32_bwd) and the flow standardisation of preprocess_flow_batch (cis_flow_stats + cis_flow_standardize,
cis_flow_standardize_bwd).  Each row reports the time per call and the achieved bytes/s -- the bytes the op must move at least (every
input element read once, every output element written once) over the measured time -- against the H100 SXM's 3.35 TB/s of HBM3.
The card's name and power limit are read in the same run.

    python tools/time_layer_ops.py [--iters 200] [--json OUT.json]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from unsupervised_detection_b200 import _lib  # noqa: E402

PEAK_BW = 3.35e12


def card():
    try:
        out = subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'], text=True)
        return out.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name(0) + ', power limit unknown'


def time_call(fn, iters):
    for _ in range(10):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e-3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=200)
    ap.add_argument('--json', default='')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'time_layer_ops.py measures on the GPU'
    lib = _lib.load()
    st = torch.cuda.current_stream().cuda_stream
    rows = []

    def row(name, shape, nbytes, fn):
        t = time_call(fn, args.iters)
        rows.append(dict(op=name, shape=shape, us=t * 1e6, GBps=nbytes / t / 1e9, frac_peak=nbytes / t / PEAK_BW))

    cases = [((4, 128, 224, 64), (256, 448), 'x2 up'), ((4, 384, 640, 2), (256, 448), 'down')]
    for (N, H, W, C), (OH, OW), what in cases:
        x = torch.randn(N, H, W, C, device='cuda')
        y = torch.empty(N, OH, OW, C, device='cuda')
        dx = torch.empty_like(x)
        nbytes = 4 * (x.numel() + y.numel())
        for method, mname in ((_lib.RESIZE_BILINEAR, 'bilinear'), (_lib.RESIZE_NEAREST, 'nearest')):
            for ac in (0, 1):
                tag = '%s ac=%d %s' % (mname, ac, what)
                shape = '[%d,%d,%d,%d] -> %dx%d' % (N, H, W, C, OH, OW)
                row('resize fwd ' + tag, shape, nbytes, lambda: lib.cis_resize_f32(x.data_ptr(), N, H, W, C, y.data_ptr(), OH, OW, method, ac, st))
                row('resize bwd ' + tag, shape, nbytes,
                    lambda: lib.cis_resize_f32_bwd(y.data_ptr(), N, OH, OW, C, H, W, dx.data_ptr(), method, ac, st))
    B, H, W = 4, 384, 640
    f = torch.randn(B, H, W, 2, device='cuda')
    out, g, dxf = torch.empty_like(f), torch.randn_like(f), torch.empty_like(f)
    stats = torch.zeros(B, 4, dtype=torch.float64, device='cuda')
    scratch = torch.empty(B * 256, dtype=torch.float64, device='cuda')

    def std_fwd():
        lib.cis_zero(stats.data_ptr(), stats.numel() * 8, st)
        lib.cis_flow_stats(f.data_ptr(), B, H * W, stats.data_ptr(), st)
        lib.cis_flow_standardize(f.data_ptr(), stats.data_ptr(), B, H * W, out.data_ptr(), st)
    n = f.numel() * 4
    row('flow standardise fwd (stats + normalise)', '[4,384,640,2]', 2 * n, std_fwd)
    row('flow standardise bwd (sums + dx)', '[4,384,640,2]', 3 * n,
        lambda: lib.cis_flow_standardize_bwd(out.data_ptr(), g.data_ptr(), stats.data_ptr(), B, H * W, scratch.data_ptr(), dxf.data_ptr(), st))
    torch.cuda.synchronize()
    c = card()
    print('card: %s' % c)
    for r in rows:
        print('%-44s %-26s %9.1f us %8.1f GB/s %5.1f %% of 3.35 TB/s' % (r['op'], r['shape'], r['us'], r['GBps'], 100 * r['frac_peak']))
    if args.json:
        with open(args.json, 'w') as fh:
            json.dump(dict(card=c, rows=rows), fh, indent=1)


if __name__ == '__main__':
    main()
