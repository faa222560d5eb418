"""Time the PWC-Net training step (FlowTrainGraph: PWC-Net forward -> multi-scale loss -> full backward -> TF-Adam + L2 -> re-pack, replayed
as CUDA graphs, as train_flow.py runs it) at 384x640, batch 8, for the tfoptflow 'lg' network (dense connections, context network) and the
'sm' one (no dense connections).

The two networks are timed in alternation inside one process (--rounds rounds, CUDA events, warm-up first), so that clock and thermal drift
hit both alike.  Prints the card's name and power limit, one JSON line per network and round, then the medians in ms/step and
frame-pairs/s, and the peak device memory of each network's step.

--flow_loss unsupervised times the 'lg' network's unsupervised step (census + smoothness, the network on both directions of each pair)
against its multi-scale step instead, alternated the same way, and then, in a separate torch.profiler run, the kernels of
cis_unsup_flow_loss and cis_unsup_flow_loss_bwd against their HBM byte roofline (bytes per pixel from the shapes, unsup_bytes below).

--flow_aug times the 'lg' network's multi-scale step with and without the augmentation of its batch (FlowTrainGraph(augment=True)),
alternated the same way, and then, in a separate torch.profiler run, cis_flow_augment's kernel against its HBM byte roofline (AUG_BYTES).
Usage: python tools/time_flow_train.py [--flow_loss multiscale|unsupervised] [--flow_aug] [--rounds 5] [--steps 20] [--warmup 5]"""
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
HBM_TBS = 3.35                                       # H100 SXM data-sheet HBM3 bandwidth
# HBM bytes per output pixel of one sample that cis_flow_augment must move, each element read or written once (the bilinear corners come
# from cache): fp32 img1, img2 [3] and gt [2] read, the same written
AUG_BYTES = 4 * (3 + 3 + 2) * 2


def unsup_bytes():
    """HBM bytes per pixel of each direction (2B x H x W pixels) that the unsupervised loss kernels must move, each tensor element read or
    written once (neighbours and bilinear corners come from cache): fp32 flow [2], frames [3], T~, M, k [1], dflow [2]."""
    return {'unsup_warp_mask_kernel': 4 * (2 + 2 + 3 + 1 + 1),      # own flow, partner flow, T, -> T~, M
            'unsup_census_kernel': 4 * (3 + 1 + 1 + 2 + 1),         # S, T~, M, flow -> k
            'unsup_bwd_kernel': 4 * (3 + 1 + 1 + 2 + 3 + 2)}        # S, T~, k, flow, T -> dflow


class Case(object):
    def __init__(self, name, options, seed=0, loss='multiscale', augment=False):
        self.name = name
        base = torch.cuda.memory_allocated()               # the networks built before this one
        torch.cuda.reset_peak_memory_stats()
        self.graph = g = FlowTrainGraph(H, W, B, options=options, loss=loss, augment=augment)
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


def profile_kernels(case, per, npix, steps=5):
    """{kernel name: [device times, us]} of the kernels named in `per` over `steps` eager steps under torch.profiler; printed against
    their byte roofline (per[k] bytes per pixel, npix pixels)."""
    from torch.profiler import ProfilerActivity, profile
    g = case.graph
    for _ in range(2):
        g.train_step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            g.train_step()
        torch.cuda.synchronize()
    times = {}
    for e in prof.events():
        for k in per:
            if k in e.name:
                times.setdefault(k, []).append(e.device_time_total if hasattr(e, 'device_time_total') else e.cuda_time_total)
    for k, b in per.items():
        t = times.get(k)
        if not t:
            print('  %-24s not found in the trace' % k)
            continue
        us = sum(t) / len(t)
        byte = b * npix
        floor = byte / (HBM_TBS * 1e12) * 1e6
        print(json.dumps(dict(kernel=k, us=round(us, 1), mbytes=round(byte / 1e6, 1), roofline_us=round(floor, 1),
                              share_of_bw_roofline=round(floor / us, 3))))


def profile_unsup(case, steps=5):
    print('unsupervised loss kernels (%d directions x %dx%d, mean of %d launches each, torch.profiler):' % (2 * B, H, W, steps))
    profile_kernels(case, unsup_bytes(), 2 * B * H * W, steps)


def profile_aug(case, steps=5):
    print('augmentation kernel (%d samples x %dx%d, mean of %d launches, torch.profiler):' % (B, H, W, steps))
    profile_kernels(case, {'flow_augment_kernel': AUG_BYTES}, B * H * W, steps)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--flow_loss', default='multiscale', choices=['multiscale', 'unsupervised'])
    ap.add_argument('--flow_aug', action='store_true', help='time the multi-scale step with and without augmentation')
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    print('card: %s' % card())
    print('PWC-Net training step %dx%d batch %d, CUDA graphs; %d rounds x %d steps (warm-up %d)' % (H, W, B, args.rounds, args.steps, args.warmup))
    if args.flow_aug:
        cases = [Case('lg-multiscale', None), Case('lg-multiscale-aug', None, augment=True)]
    elif args.flow_loss == 'unsupervised':
        cases = [Case('lg-multiscale', None), Case('lg-unsup', None, loss='unsupervised')]
    else:
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
    if args.flow_aug:
        profile_aug(cases[1])
    elif args.flow_loss == 'unsupervised':
        profile_unsup(cases[1])


if __name__ == '__main__':
    main()
