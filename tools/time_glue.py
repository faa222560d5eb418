"""Warm per-launch time of every non-convolution launch of the train step, set against the HBM byte roofline.

Same method as tools/time_ops.py: each launch of fwd, bwd['G'] and bwd['R'] is captured REPS times back to back in a CUDA graph and
replayed after one untimed run, so L2 stays warm as in the real step and host-side launch cost is excluded.  Bytes come from the launch
arguments (bytes_of below): every element a kernel must read or write counted once, so a launch's roofline fraction is
bytes / peak / time.  The peak is MEASURED_PEAKS.json's hbm_gbs when that file is present, else the 3.35 TB/s H100 SXM data-sheet
figure.  Per-step sums weight fwd x4, bwd['G'] x3 and bwd['R'] x1 and divide by 4 (one 1R:3G cycle is four steps).

  python tools/time_glue.py                         # table on stdout
  TIME_GLUE_JSON=out.json python tools/time_glue.py # plus one JSON row per launch
"""
import collections
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from unsupervised_detection_b200.common_flags import Config
from unsupervised_detection_b200.models.adversarial_learner import AdversarialLearner

REPS = 20
CONV = ('cis_conv_igemm', 'cis_conv_wgrad')


def peak_gbs():
    path = os.path.join(ROOT, 'MEASURED_PEAKS.json')
    if os.path.exists(path):
        return float(json.load(open(path))['hbm_gbs']), 'measured'
    return 3350.0, 'data sheet'


def bytes_of(name, a):
    """Bytes a launch must move, from its arguments (None for launches without a formula here)."""
    if name == 'cis_dact_colsum':      # g, y, y_pitch, ..., res, ..., npix, nch, act, alpha, part, nblocks
        npix, nch, nblk = a[9], a[10], a[14]
        return npix * (-(-nch // 8)) * 16 * (3 + (a[6] is not None)) + 4 * nblk * nch
    if name == 'cis_dact_mul':         # g read + written, y read, res read
        npix, chunks = a[9], a[10]
        return npix * chunks * 16 * (3 + (a[6] is not None))
    if name == 'cis_colsum':           # g read, partials written
        npix, nch, nblk = a[3], a[4], a[6]
        return npix * (-(-nch // 8)) * 16 + 4 * nblk * nch
    if name == 'cis_add_slice':        # reps sources read, dst read when accumulating, dst written
        npix, chunks, reps, acc = a[6], a[7], a[8], a[9]
        return npix * chunks * 16 * (reps + 1 + (1 if acc else 0))
    if name == 'cis_resize_concat_bf16_bwd':   # ddst slices of the wanted sources read once, each gradient written (read if accumulated)
        grads, want, acc, nsrc, N, OH, OW, H, W = a[6], a[7], a[8], a[9], a[3], a[4], a[5], a[10], a[11]
        b = 0
        for i in range(nsrc):
            if want[i]:
                rows = grads[i].n_mod or N
                b += grads[i].chunks * 16 * (N * OH * OW + rows * H * W * (2 if acc[i] else 1))
        return b
    if name == 'cis_upsample_nn2x_bwd':        # ddst (N, 2H, 2W, pitch) read, dsrc (N, H, W, pitch) written (read if accumulated)
        N, H, W, pitch, acc = a[1], a[2], a[3], a[4], a[6]
        return 2 * pitch * N * H * W * (4 + 1 + (1 if acc else 0))
    if name == 'cis_resize_f32_bwd_to_bf16':   # fp32 ddst read, C bf16 channels of dsrc written
        N, OH, OW, C, H, W = a[1:7]
        return 4 * N * OH * OW * C + 2 * N * H * W * C
    if name == 'cis_resize_concat_bf16':       # sources read once, destination slice written
        srcs, nsrc, N, H, W, OH, OW = a[0], a[1], a[2], a[3], a[4], a[8], a[9]
        return sum(srcs[i].chunks * 16 * ((srcs[i].n_mod or N) * H * W + N * OH * OW) for i in range(nsrc))
    if name == 'cis_zero':
        return a[1]
    return None


def time_launch(fn, a, st):
    fn(*a, st.cuda_stream)
    torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        cs = torch.cuda.current_stream().cuda_stream
        for _ in range(REPS):
            fn(*a, cs)
    gr.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    gr.replay()
    e1.record()
    torch.cuda.synchronize()
    del gr
    return e0.elapsed_time(e1) * 1e3 / REPS


def main():
    assert torch.cuda.is_available(), 'time_glue.py times launches on a CUDA device'
    L = AdversarialLearner()
    L.config = Config(img_height=256, img_width=448, batch_size=4, dataset='SYNTHETIC', flow_ckpt='synthetic', summary_freq=10 ** 9)
    L.build_train_graph()
    b = L.reader.batch(4)
    L.feed(b[0], b[1])
    g = L.graph
    for m in 'GR':
        g.train_step(m)
    torch.cuda.synchronize()
    st = torch.cuda.current_stream()
    pk, pk_src = peak_gbs()
    rows = []
    for pname, plan, w in (('fwd', g.fwd, 4), ('bwdG', g.bwd['G'], 3), ('bwdR', g.bwd['R'], 1)):
        for i, (fn, a, name, _, lane) in enumerate(plan.ops):
            if fn is None or name in CONV:
                continue
            us = time_launch(fn, a, st)
            nb = bytes_of(name, a)
            rows.append(dict(plan=pname, idx=i, w=w, op=name, lane=lane, us=us, bytes=nb,
                             frac=(nb / (pk * 1e3) / us) if nb is not None and us > 0 else None))
    if os.environ.get('TIME_GLUE_JSON'):
        json.dump(rows, open(os.environ['TIME_GLUE_JSON'], 'w'))
    print('device %s, peak %.0f GB/s (%s), %d reps per launch' % (torch.cuda.get_device_name(), pk, pk_src, REPS))
    print('%-5s %4s %-30s %4s %9s %9s %7s' % ('plan', 'idx', 'op', 'lane', 'us', 'MB', 'roof'))
    for r in rows:
        print('%-5s %4d %-30s %4d %9.2f %9s %7s' % (r['plan'], r['idx'], r['op'], r['lane'], r['us'],
                                                   '-' if r['bytes'] is None else '%.2f' % (r['bytes'] / 1e6),
                                                   '-' if r['frac'] is None else '%.0f%%' % (100 * r['frac'])))
    agg = collections.defaultdict(lambda: [0.0, 0.0, 0.0, True])
    for r in rows:
        k = agg[r['op']]
        k[0] += r['w'] / 4.0
        k[1] += r['w'] * r['us'] / 4.0
        if r['bytes'] is None:
            k[3] = False
        else:
            k[2] += r['w'] * r['bytes'] / 4.0
    print('--- per step (1R:3G weighted)')
    print('%-30s %7s %10s %9s %7s' % ('op', 'n/step', 'us/step', 'MB/step', 'roof'))
    for name, (n, us, nb, full) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print('%-30s %7.2f %10.1f %9s %7s' % (name, n, us, '%.1f' % (nb / 1e6) if full else '-',
                                             '%.0f%%' % (100 * nb / (pk * 1e3) / us) if full and us > 0 else '-'))
    print('non-conv launches: %.1f us/step' % sum(v[1] for v in agg.values()))


if __name__ == '__main__':
    main()
