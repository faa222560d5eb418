"""Warm per-launch timing of every op of the step (CUDA events on the launching stream, each op replayed REPS times back to back
after one untimed run).  Unlike the ncu launch list (cold caches, serialised) this keeps L2 warm like the real step."""
import os, sys, json, collections
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from unsupervised_detection_b200 import engine
from unsupervised_detection_b200.common_flags import Config
from unsupervised_detection_b200.models.adversarial_learner import AdversarialLearner

REPS = 10
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
rows = []
for pname, plan, w in (('fwd', g.fwd, 4), ('bwdG', g.bwd['G'], 3), ('bwdR', g.bwd['R'], 1)):
    for i, (fn, a, name, fl, lane) in enumerate(plan.ops):
        if fn is None:
            continue
        # replay through a CUDA graph so host-side launch cost (descriptor checks, tensor-map encodes) is excluded
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
        us = e0.elapsed_time(e1) * 1e3 / REPS
        del gr
        info = ''
        if name == 'cis_conv_igemm':
            d = a[0]._obj
            info = '%s BN%d MT%d N%d %dx%d taps%d ch%d sp%d' % ('halo' if d.halo else 'gen', d.BN, d.MT, d.N, d.OH, d.OW, d.ntaps,
                                                               sum(d.src[k].chunks for k in range(d.nsrc)) * 8, d.splits)
        elif name == 'cis_conv_wgrad':
            d = a[0]._obj
            info = 'tma%d N%d %dx%d taps%d cout%d K%d sp%d' % (d.tma, d.N, d.OH, d.OW, d.ntaps, d.Cout, d.K_pad, d.splits)
            if d.tma == 2:
                info += ' nh%d nwg%d' % (d.nh or 64, max(d.nwg, 1))
        rows.append((pname, w, name, us, fl, info))
if os.environ.get('TIME_OPS_JSON'):
    # one row per launch, keyed by (plan, index-in-plan): lets tools/ab_diff.py line up the same layer across two configurations
    json.dump([dict(plan=p, w=w, op=n, us=us, flops=fl, info=info) for p, w, n, us, fl, info in rows], open(os.environ['TIME_OPS_JSON'], 'w'))
tot = sum(r[1] * r[3] for r in rows) / 4
print('sum of warm per-op times per step: %.1f us' % tot)
agg = collections.defaultdict(lambda: [0, 0.0, 0.0])
for p, w, n, us, fl, info in rows:
    k = n + (' halo' if info.startswith('halo') else ' gen' if info.startswith('gen') else '')
    agg[k][0] += w / 4.0; agg[k][1] += w * us / 4; agg[k][2] += w * fl / 4
for k, v in sorted(agg.items(), key=lambda kv: -kv[1][1]):
    print('%-34s n/step %6.1f  %8.1f us/step  %6.1f%%  %s' % (k, v[0], v[1], 100 * v[1] / tot, ('%.0f TF/s' % (v[2] / v[1] / 1e6)) if v[2] else ''))
print('--- all conv ops by weighted time')
for p, w, n, us, fl, info in sorted([r for r in rows if 'conv' in r[2]], key=lambda r: -r[1] * r[3]):
    print('%-5s x%d %-18s %8.1f us %7.1f GF %6.0f TF/s  %s' % (p, w, n[4:], us, fl / 1e9, fl / us / 1e6 if us else 0, info))
small = [r for r in rows if r[2] == 'cis_conv_igemm' and r[3] < 15]
print('conv launches < 15 us: n/step %.0f, us/step %.0f' % (sum(r[1] for r in small) / 4, sum(r[1] * r[3] for r in small) / 4))
