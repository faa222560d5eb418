"""Time the PWC-Net training step (FlowTrainGraph: PWC-Net forward -> multi-scale loss -> full backward -> TF-Adam + L2 -> re-pack, replayed
as CUDA graphs, as train_flow.py runs it) at 384x640, batch 8, for the tfoptflow 'lg' network (dense connections, context network) and the
'sm' one (no dense connections).

The two networks are timed in alternation inside one process (--rounds rounds, CUDA events, warm-up first), so that clock and thermal drift
hit both alike.  Prints the card's name and power limit, one JSON line per network and round, then the medians in ms/step and
frame-pairs/s, and the peak device memory of each network's step.
Usage: python tools/time_flow_train.py [--rounds 5] [--steps 20] [--warmup 5]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.time_pwc_options import card, timed_ms  # noqa: E402
from unsupervised_detection_b200 import params_init  # noqa: E402
from unsupervised_detection_b200.flow_train_graph import FlowTrainGraph  # noqa: E402

B, H, W = 8, 384, 640
NETS = {'lg': None, 'sm': {'use_dense_cx': False}}


class Case(object):
    def __init__(self, name, options, seed=0):
        self.name = name
        base = torch.cuda.memory_allocated()               # the networks built before this one
        torch.cuda.reset_peak_memory_stats()
        self.graph = g = FlowTrainGraph(H, W, B, options=options)
        g.load_params(params_init.init_pwcnet(g.store.entries))
        gen = torch.Generator().manual_seed(seed)
        a = torch.rand(B, H, W, 3, generator=gen) - 0.5
        g.feed(a.cuda(), torch.roll(a, shifts=(2, 3), dims=(1, 2)).cuda(), torch.full((B, H, W, 2), -2.5).cuda())
        g.train_step(use_graph=True)
        torch.cuda.synchronize()
        self.peak_gb = (torch.cuda.max_memory_allocated() - base) / 2 ** 30

    def step(self, _):
        self.graph.train_step(use_graph=True)

    def measure(self, steps, warmup):
        timed_ms(self.step, warmup)
        ms = timed_ms(self.step, steps)
        return dict(step_ms=ms, pairs_per_s=B / (ms / 1e3))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    print('card: %s' % card())
    print('PWC-Net training step %dx%d batch %d, CUDA graphs; %d rounds x %d steps (warm-up %d)' % (H, W, B, args.rounds, args.steps, args.warmup))
    cases = [Case(n, o) for n, o in NETS.items()]
    for c in cases:
        print(json.dumps(dict(graph=c.name, launches_per_step=c.graph.launches_per_step(), params=c.graph.store.real_count(),
                              peak_mem_gb_after_build_and_first_step=round(c.peak_gb, 2))))
    rows = {c.name: [] for c in cases}
    for r in range(args.rounds):
        for c in cases:
            m = c.measure(args.steps, args.warmup)
            rows[c.name].append(m)
            print(json.dumps(dict(graph=c.name, round=r, **{k: round(v, 3) for k, v in m.items()})))
            sys.stdout.flush()
    med = lambda v: sorted(v)[len(v) // 2]
    print('medians over %d rounds:' % args.rounds)
    for n in rows:
        s = {k: med([m[k] for m in rows[n]]) for k in rows[n][0]}
        print('  %-3s %7.2f ms/step  %6.1f frame-pairs/s' % (n, s['step_ms'], s['pairs_per_s']))


if __name__ == '__main__':
    main()
