"""What the moving average of the weights (--ema_decay) costs on the GPU.

  cis    the CIS train step at bench.py's shape (256x448, batch 4, PWC-Net at 384x640 in the loop, CUDA graphs, the pipelined schedule,
         1 recover : 3 generator steps), averaging off and on
  flow   the PWC-Net training step at train_flow.py's defaults (192x384, batch 16, frames uploaded at 384x640), off and on
  ema    cis_ema_update alone on each trained store (generator, recover net, PWC-Net): time per launch over --launches launches, and the
         achieved rate of its 12 bytes per parameter (read shadow and param, write shadow) against the 3.35 TB/s of the H100 SXM data sheet.
         The launches cycle over enough (shadow, param) pairs to fill 256 MB, five times the 50 MB L2, so each one streams from HBM;
         inside a train step the recover net's 41 MB may partly hit L2 instead

The off and on graphs of each pair are timed in alternation inside one process (--rounds rounds, CUDA events, warm-up first), so that clock
drift hits both alike.  Prints the card's name and power limit, one JSON line per measurement, then the medians.
Usage: python tools/time_ema.py [--rounds 5] [--steps 40] [--warmup 8] [--launches 200]"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.time_pwc_options import card, timed_ms  # noqa: E402
from unsupervised_detection_b200 import _lib, params_init  # noqa: E402
from unsupervised_detection_b200.flow_train_graph import FlowTrainGraph  # noqa: E402
from unsupervised_detection_b200.models.PWCNet.model_pwcnet import _DEFAULT_PWCNET_TEST_OPTIONS  # noqa: E402
from unsupervised_detection_b200.step_graph import CISGraph  # noqa: E402

DECAY = 0.999
HBM_TBS = 3.35                                       # H100 SXM data-sheet HBM3 bandwidth


class CisCase(object):
    def __init__(self, decay):
        self.g = g = CISGraph(256, 448, 4, with_pwc=True, pwc_options=_DEFAULT_PWCNET_TEST_OPTIONS, ema_decay=decay)
        p = params_init.init_generator()
        p.update(params_init.init_recover())
        p.update(params_init.init_pwcnet(g.pwc_store.entries))
        g.load_params(p)
        gen = torch.Generator().manual_seed(0)
        a = torch.rand(4, 384, 640, 3, generator=gen) - 0.5
        g.feed(a.cuda(), torch.roll(a, shifts=(2, 3), dims=(1, 2)).cuda())
        self.k = 0

    def step(self, _):
        self.k += 1
        self.g.train_step('R' if self.k % 4 == 0 else 'G', use_graph=True, pipeline=True)


class FlowCase(object):
    def __init__(self, decay):
        self.g = g = FlowTrainGraph(192, 384, 16, options=_DEFAULT_PWCNET_TEST_OPTIONS, in_hw=(384, 640), ema_decay=decay)
        g.load_params(params_init.init_pwcnet(g.store.entries))
        gen = torch.Generator().manual_seed(0)
        a = torch.rand(16, 384, 640, 3, generator=gen) - 0.5
        g.feed(a.cuda(), torch.roll(a, shifts=(2, 3), dims=(1, 2)).cuda(), torch.full((16, 384, 640, 2), -2.5).cuda())

    def step(self, _):
        self.g.train_step(use_graph=True)


def alternate(name, make, args):
    cases = {'off': make(0.0), 'on': make(DECAY)}
    for c in cases.values():
        timed_ms(c.step, args.warmup)
    ms = {k: [] for k in cases}
    for r in range(args.rounds):
        for k, c in cases.items():
            ms[k].append(timed_ms(c.step, args.steps))
            print(json.dumps({'case': name, 'ema': k, 'round': r, 'step_ms': round(ms[k][-1], 4)}))
    med = {k: statistics.median(v) for k, v in ms.items()}
    print('%-5s step median: off %.3f ms, on %.3f ms, difference %+.3f ms (%+.2f %%)'
          % (name, med['off'], med['on'], med['on'] - med['off'], 100 * (med['on'] / med['off'] - 1)))
    for c in cases.values():
        c.g.graphs.clear()
    del cases
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def ema_alone(args):
    sizes = {}
    g = CISGraph(256, 448, 4, with_pwc=True, pwc_options=_DEFAULT_PWCNET_TEST_OPTIONS, train=False, device='cpu')
    sizes.update(generator=g.gen_store.size, recover=g.rec_store.size, pwcnet=g.pwc_store.size)
    step = torch.full((1,), 100, dtype=torch.int64, device='cuda')
    st = torch.cuda.current_stream().cuda_stream
    for name, n in sizes.items():
        pairs = [(torch.randn(n, device='cuda'), torch.randn(n, device='cuda')) for _ in range(-(-(256 << 20) // (8 * n)))]

        def launch(i):
            shadow, param = pairs[i % len(pairs)]
            _lib.call('cis_ema_update', shadow.data_ptr(), param.data_ptr(), n, DECAY, step.data_ptr(), st)
        timed_ms(launch, 20)
        us = [1e3 * timed_ms(launch, args.launches) for _ in range(args.rounds)]
        t = statistics.median(us)
        gbs = 12 * n / (t * 1e-6) / 1e9
        print(json.dumps({'case': 'ema', 'store': name, 'params': n, 'buffers': len(pairs), 'us_per_launch': round(t, 2),
                          'GB_s': round(gbs, 1), 'of_hbm_datasheet': round(gbs / (HBM_TBS * 1e3), 3)}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--steps', type=int, default=40)
    ap.add_argument('--warmup', type=int, default=8)
    ap.add_argument('--launches', type=int, default=200)
    args = ap.parse_args()
    print('card: %s' % card())
    ema_alone(args)
    alternate('cis', CisCase, args)
    alternate('flow', FlowCase, args)


if __name__ == '__main__':
    main()
