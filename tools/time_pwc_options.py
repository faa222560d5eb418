"""Time the PWC-Net option sets on one GPU: the function-level forward (ModelPWCNet(options=...).predict_from_img_pairs at 384x640,
batch 4) and the 256x448 batch-4 train step through CISGraph(pwc_options=...), with the frozen flow network both pipelined (as the
training loop and bench.py run it: the flow network of the next batch overlaps the current step on a second stream) and sequential.

The option sets are timed in alternation inside one process (round-robin over --rounds rounds, CUDA events, warm-up first), so that clock
and thermal drift hit every set alike.  Prints the card's name and power limit, one JSON line per set and round, then the medians.
Usage: python tools/time_pwc_options.py [--sets lg,sm,lg_nores,sm_nores,lg_r3] [--rounds 3] [--steps 20] [--warmup 4]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from unsupervised_detection_b200 import params_init  # noqa: E402
from unsupervised_detection_b200.models.PWCNet.model_pwcnet import ModelPWCNet, _DEFAULT_PWCNET_TEST_OPTIONS  # noqa: E402
from unsupervised_detection_b200.step_graph import CISGraph  # noqa: E402

SETS = {
    'lg': {},
    'sm': {'use_dense_cx': False},
    'lg_nores': {'use_res_cx': False},
    'sm_nores': {'use_dense_cx': False, 'use_res_cx': False},
    'lg_r3': {'search_range': 3},
}
FWD_B, FWD_H, FWD_W = 4, 384, 640
TR_B, TR_H, TR_W = 4, 256, 448
ITERS_REC, ITERS_GEN = 1, 3          # common_flags defaults: one recover step, then three generator steps


def card():
    q = 'name,power.limit,clocks.max.sm'
    try:
        o = subprocess.run(['nvidia-smi', '-i', str(torch.cuda.current_device()), '--query-gpu=' + q, '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception as e:      # nvidia-smi missing: the name from the driver, the power limit unknown
        o = '%s, unknown (%s)' % (torch.cuda.get_device_name(), type(e).__name__)
    return o


def timed_ms(fn, k):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(k):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / k


class Case(object):
    def __init__(self, name, over, seed=0):
        self.name = name
        self.options = dict(_DEFAULT_PWCNET_TEST_OPTIONS, **over)
        self.model = ModelPWCNet(options=self.options)
        g = torch.Generator().manual_seed(seed)
        self.a = (torch.rand(FWD_B, FWD_H, FWD_W, 3, generator=g) - 0.5).cuda()
        self.b = torch.roll(self.a, shifts=(2, 3), dims=(1, 2))
        self.graph = CISGraph(TR_H, TR_W, TR_B, pwc_options=self.options)
        p = {}
        p.update(params_init.init_generator())
        p.update(params_init.init_recover())
        p.update(params_init.init_pwcnet(self.graph.pwc_store.entries))
        self.params = {k: v for k, v in p.items() if k.startswith('pwcnet/')}
        self.params = {k: v.cuda() for k, v in self.params.items()}
        self.graph.load_params(p)
        self.graph.img1.copy_(self.a)
        self.graph.img2.copy_(self.b)
        self.n = 0

    def forward(self, _):
        self.model.predict_from_img_pairs(self.a, self.b, params=self.params)

    def step(self, pipeline):
        def one(_):
            self.n += 1
            mode = 'R' if self.n % (ITERS_REC + ITERS_GEN) < ITERS_REC else 'G'
            self.graph.train_step(mode, use_graph=True, pipeline=pipeline)
        return one

    def measure(self, steps, warmup):
        out = {}
        with torch.no_grad():
            timed_ms(self.forward, warmup)
            out['fwd_ms'] = timed_ms(self.forward, steps)
        for pipe, key in ((True, 'step_pipelined_ms'), (False, 'step_sequential_ms')):
            timed_ms(self.step(pipe), warmup)
            out[key] = timed_ms(self.step(pipe), steps)
            self.graph.pipeline_drain()
        out['fwd_pairs_per_s'] = FWD_B / (out['fwd_ms'] / 1e3)
        out['step_pipelined_pairs_per_s'] = TR_B / (out['step_pipelined_ms'] / 1e3)
        out['step_sequential_pairs_per_s'] = TR_B / (out['step_sequential_ms'] / 1e3)
        return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--sets', default='lg,sm', help='comma-separated subset of ' + ','.join(SETS))
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=4)
    args = ap.parse_args()
    names = args.sets.split(',')
    for n in names:
        if n not in SETS:
            raise SystemExit('unknown set %r (known: %s)' % (n, ', '.join(SETS)))
    torch.cuda.set_device(0)
    print('card: %s' % card())
    print('forward %dx%d batch %d; train step %dx%d batch %d; %d rounds x %d steps (warm-up %d)'
          % (FWD_H, FWD_W, FWD_B, TR_H, TR_W, TR_B, args.rounds, args.steps, args.warmup))
    cases = [Case(n, SETS[n]) for n in names]
    rows = {n: [] for n in names}
    for r in range(args.rounds):
        for c in cases:
            m = c.measure(args.steps, args.warmup)
            rows[c.name].append(m)
            print(json.dumps(dict(set=c.name, round=r, **{k: round(v, 3) for k, v in m.items()})))
            sys.stdout.flush()
    med = lambda v: sorted(v)[len(v) // 2]
    print('medians over %d rounds:' % args.rounds)
    for n in names:
        s = {k: med([m[k] for m in rows[n]]) for k in rows[n][0]}
        print('  %-9s fwd %7.2f ms (%6.1f pairs/s)  step pipelined %6.2f ms (%6.1f pairs/s)  sequential %6.2f ms (%6.1f pairs/s)'
              % (n, s['fwd_ms'], s['fwd_pairs_per_s'], s['step_pipelined_ms'], s['step_pipelined_pairs_per_s'], s['step_sequential_ms'],
                 s['step_sequential_pairs_per_s']))


if __name__ == '__main__':
    main()
