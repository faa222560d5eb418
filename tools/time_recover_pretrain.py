"""Time the recover-net pretraining step (CISGraph(masks='boxes'): PWC-Net -> box masks -> 3x recover -> losses -> backward -> clip + Adam)
against the recover step of the adversarial graph (the same step with the generator's forward in front of it), both at 256x448, batch 4,
PWC-Net at 384x640, with the frozen flow network pipelined as pretrain_recover.py and train.py run it.

The two graphs are timed in alternation inside one process (--rounds rounds, CUDA events, warm-up first), so that clock and thermal drift hit
both alike.  Prints the card's name and power limit, one JSON line per graph and round, then the medians in frame-pairs/s.
--flow gt times the pretraining step on ground-truth flow (CISGraph(flow_source='input'): no PWC-Net, the flow is uploaded at 384x640)
against the same step on PWC-Net's flow instead.
Usage: python tools/time_recover_pretrain.py [--flow pwc|gt] [--rounds 5] [--steps 30] [--warmup 5]"""
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
    def __init__(self, name, masks, seed=0, flow_source='pwc'):
        self.name = name
        self.graph = CISGraph(H, W, B, masks=masks, flow_source=flow_source)
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

    def step(self, _):
        self.graph.train_step('R', use_graph=True, pipeline=True)

    def measure(self, steps, warmup):
        timed_ms(self.step, warmup)
        ms = timed_ms(self.step, steps)
        self.graph.pipeline_drain()
        return dict(step_ms=ms, pairs_per_s=B / (ms / 1e3))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--flow', choices=['pwc', 'gt'], default='pwc', help='gt: ground-truth flow pretraining vs PWC-Net flow pretraining')
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--steps', type=int, default=30)
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    print('card: %s' % card())
    print('recover step %dx%d batch %d, PWC-Net 384x640, pipelined; %d rounds x %d steps (warm-up %d)'
          % (H, W, B, args.rounds, args.steps, args.warmup))
    if args.flow == 'gt':
        cases = [Case('pretrain_gt_flow', 'boxes', flow_source='input'), Case('pretrain_boxes', 'boxes')]
    else:
        cases = [Case('pretrain_boxes', 'boxes'), Case('adversarial_R', 'generator')]
    a, b = (c.name for c in cases)
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
        print('  %-17s %6.2f ms/step  %7.1f frame-pairs/s' % (n, s[n]['step_ms'], s[n]['pairs_per_s']))
    print('  %s / %s throughput: %.3f' % (a, b, s[a]['pairs_per_s'] / s[b]['pairs_per_s']))
    if args.flow == 'gt':
        validation_share(args.steps, args.warmup)


def validation_share(steps, warmup):
    """One batch of validate_recover on ground-truth flow (eager forward of a forward-only boxes graph + cis_masked_epe) against
    cis_masked_epe alone: the EPE kernel's share of a validation pass."""
    g = CISGraph(H, W, B, masks='boxes', flow_source='input', train=False)
    g.load_params(dict(params_init.init_generator(), **params_init.init_recover()))
    g.flow_full.normal_(0.0, 3.0)

    def batch(_):
        g.forward()
        g.masked_epe()
    timed_ms(batch, warmup)
    full = timed_ms(batch, steps)
    timed_ms(lambda _: g.masked_epe(), warmup)
    epe = timed_ms(lambda _: g.masked_epe(), steps)
    print(json.dumps(dict(graph='validate_gt_flow', batch_ms=round(full, 4), masked_epe_ms=round(epe, 4), epe_share=round(epe / full, 4))))


if __name__ == '__main__':
    main()
