"""Time the recover-net pretraining step (CISGraph(masks='boxes'): PWC-Net -> box masks -> 3x recover -> losses -> backward -> clip + Adam)
against the recover step of the adversarial graph (the same step with the generator's forward in front of it), both at 256x448, batch 4,
PWC-Net at 384x640, with the frozen flow network pipelined as pretrain_recover.py and train.py run it.

The two graphs are timed in alternation inside one process (--rounds rounds, CUDA events, warm-up first), so that clock and thermal drift hit
both alike.  Prints the card's name and power limit, one JSON line per graph and round, then the medians in frame-pairs/s.
Usage: python tools/time_recover_pretrain.py [--rounds 5] [--steps 30] [--warmup 5]"""
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
    def __init__(self, name, masks, seed=0):
        self.name = name
        self.graph = CISGraph(H, W, B, masks=masks)
        p = {}
        p.update(params_init.init_generator())
        p.update(params_init.init_recover())
        p.update(params_init.init_pwcnet(self.graph.pwc_store.entries))
        self.graph.load_params(p)
        g = torch.Generator().manual_seed(seed)
        a = (torch.rand(B, 384, 640, 3, generator=g) - 0.5).cuda()
        self.graph.img1.copy_(a)
        self.graph.img2.copy_(torch.roll(a, shifts=(2, 3), dims=(1, 2)))

    def step(self, _):
        self.graph.train_step('R', use_graph=True, pipeline=True)

    def measure(self, steps, warmup):
        timed_ms(self.step, warmup)
        ms = timed_ms(self.step, steps)
        self.graph.pipeline_drain()
        return dict(step_ms=ms, pairs_per_s=B / (ms / 1e3))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--steps', type=int, default=30)
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    print('card: %s' % card())
    print('recover step %dx%d batch %d, PWC-Net 384x640, pipelined; %d rounds x %d steps (warm-up %d)'
          % (H, W, B, args.rounds, args.steps, args.warmup))
    cases = [Case('pretrain_boxes', 'boxes'), Case('adversarial_R', 'generator')]
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
        print('  %-15s %6.2f ms/step  %7.1f frame-pairs/s' % (n, s[n]['step_ms'], s[n]['pairs_per_s']))
    print('  pretraining / adversarial recover step throughput: %.3f' % (s['pretrain_boxes']['pairs_per_s'] / s['adversarial_R']['pairs_per_s']))


if __name__ == '__main__':
    main()
