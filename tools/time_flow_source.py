"""Time the adversarial train step on PWC-Net's flow (the default CISGraph) against the same step on supplied flow
(CISGraph(masks='generator', flow_source='input'): no PWC-Net, the flow is uploaded at 384x640 next to frame 1), both at 256x448,
batch 4, alternating one recover step and three generator steps (1R:3G, train.py's default), pipelined as train.py runs them.

The two graphs are timed in alternation inside one process (--rounds rounds, CUDA events, warm-up first), so that clock and thermal drift hit
both alike.  Prints the card's name and power limit, one JSON line per graph and round, then the medians in ms/step and frame-pairs/s.
Usage: python tools/time_flow_source.py [--rounds 5] [--steps 40] [--warmup 8]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.time_pwc_options import card, timed_ms  # noqa: E402
from unsupervised_detection_b200 import params_init  # noqa: E402
from unsupervised_detection_b200.step_graph import CISGraph  # noqa: E402

B, H, W = 4, 256, 448


class Case(object):
    def __init__(self, name, flow_source, seed=0):
        self.name = name
        self.graph = CISGraph(H, W, B, masks='generator', flow_source=flow_source)
        p = {}
        p.update(params_init.init_generator())
        p.update(params_init.init_recover())
        p.update(params_init.init_pwcnet(self.graph.pwc_store.entries))
        self.graph.load_params(p)
        g = torch.Generator().manual_seed(seed)
        a = (torch.rand(B, 384, 640, 3, generator=g) - 0.5).cuda()
        self.graph.img1.copy_(a)
        if flow_source == 'input':
            self.graph.flow_full.copy_(torch.randn(B, 384, 640, 2, generator=g).cuda() * 3.0)
        else:
            self.graph.img2.copy_(torch.roll(a, shifts=(2, 3), dims=(1, 2)))
        self.n = 0

    def step(self, _):
        self.graph.train_step('R' if self.n % 4 == 0 else 'G', use_graph=True, pipeline=True)
        self.n += 1

    def measure(self, steps, warmup):
        timed_ms(self.step, warmup)
        ms = timed_ms(self.step, steps)
        self.graph.pipeline_drain()
        return dict(step_ms=ms, pairs_per_s=B / (ms / 1e3))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--steps', type=int, default=40, help='a multiple of 4 keeps the 1R:3G mix exact')
    ap.add_argument('--warmup', type=int, default=8)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    print('card: %s' % card())
    print('adversarial step %dx%d batch %d, 1R:3G, pipelined; %d rounds x %d steps (warm-up %d)' % (H, W, B, args.rounds, args.steps, args.warmup))
    cases = [Case('pwc_flow', 'pwc'), Case('supplied_flow', 'input')]
    rows = {c.name: [] for c in cases}
    for r in range(args.rounds):
        for c in cases:
            m = c.measure(args.steps, args.warmup)
            rows[c.name].append(m)
            print(json.dumps(dict(graph=c.name, round=r, **{k: round(v, 3) for k, v in m.items()})))
            sys.stdout.flush()
    med = lambda v: sorted(v)[len(v) // 2]
    print('medians over %d rounds:' % args.rounds)
    s = {n: {k: med([m[k] for m in rows[n]]) for k in rows[n][0]} for n in rows}
    for n in rows:
        print('  %-14s %6.2f ms/step  %7.1f frame-pairs/s' % (n, s[n]['step_ms'], s[n]['pairs_per_s']))
    print('  supplied_flow / pwc_flow throughput: %.3f' % (s['supplied_flow']['pairs_per_s'] / s['pwc_flow']['pairs_per_s']))


if __name__ == '__main__':
    main()
