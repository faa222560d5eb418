"""What one --resumable epoch-end state write costs, as a share of an epoch.

  cis    train.py's step at bench.py's shape (256x448, batch 4, PWC-Net at 384x640 in the loop, CUDA graphs, the pipelined schedule,
         1 recover : 3 generator steps), with the generator and recover net averaged (--ema_decay): flat, m, v and shadow of both
  flow   train_flow.py's step at 384x640, batch 8, with PWC-Net averaged: the four PWC-Net buffers, about 225 MB

For each: the step time (CUDA events over --steps steps after --warmup), then the wall time of AdversarialLearner._save_train_state
(stream synchronise, device -> host copies, torch.save, fsync, rename) over --writes writes into a temporary directory, and the write's share
of one epoch at the default --num_samples_train (ceil(5000 / batch) steps).  Step time itself is unchanged by --resumable: the launch plans
do not depend on it.  Prints the card's name and power limit, one JSON line per case.
Usage: python tools/time_resume.py [--steps 40] [--warmup 8] [--writes 3]"""
import argparse
import json
import math
import os
import shutil
import statistics
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.time_pwc_options import card, timed_ms  # noqa: E402
from unsupervised_detection_b200 import params_init  # noqa: E402
from unsupervised_detection_b200.common_flags import FLAGS, Config  # noqa: E402
from unsupervised_detection_b200.data.synthetic import SyntheticReader  # noqa: E402
from unsupervised_detection_b200.flow_train_graph import FlowTrainGraph  # noqa: E402
from unsupervised_detection_b200.models.PWCNet.model_pwcnet import _DEFAULT_PWCNET_TEST_OPTIONS  # noqa: E402
from unsupervised_detection_b200.models.flow_learner import FlowLearner  # noqa: E402
from unsupervised_detection_b200.step_graph import CISGraph  # noqa: E402

DECAY = 0.999


def _learner(kind, graph, batch, ck):
    L = FlowLearner()
    L.config = Config(batch_size=batch, checkpoint_dir=ck)
    L.config.ema_decay = DECAY
    L._kind, L.graph, L.reader, L.device = kind, graph, SyntheticReader(32, 48), 'cuda:0'
    L._frozen = L._frozen_crc()
    return L


def cis(ck):
    g = CISGraph(256, 448, 4, with_pwc=True, pwc_options=_DEFAULT_PWCNET_TEST_OPTIONS, ema_decay=DECAY)
    p = params_init.init_generator()
    p.update(params_init.init_recover())
    p.update(params_init.init_pwcnet(g.pwc_store.entries))
    g.load_params(p)
    a = torch.rand(4, 384, 640, 3, generator=torch.Generator().manual_seed(0)) - 0.5
    g.feed(a.cuda(), torch.roll(a, shifts=(2, 3), dims=(1, 2)).cuda())
    return _learner('adversarial', g, 4, ck), lambda i: g.train_step('R' if i % 4 == 0 else 'G', use_graph=True, pipeline=True)


def flow(ck):
    g = FlowTrainGraph(384, 640, 8, options=_DEFAULT_PWCNET_TEST_OPTIONS, in_hw=(384, 640), ema_decay=DECAY)
    g.load_params(params_init.init_pwcnet(g.store.entries))
    a = torch.rand(8, 384, 640, 3, generator=torch.Generator().manual_seed(0)) - 0.5
    g.feed(a.cuda(), torch.roll(a, shifts=(2, 3), dims=(1, 2)).cuda(), torch.full((8, 384, 640, 2), -2.5).cuda())
    return _learner('flow', g, 8, ck), lambda i: g.train_step(use_graph=True)


def measure(name, make, args):
    ck = tempfile.mkdtemp(prefix='time_resume_')
    try:
        L, step = make(ck)
        timed_ms(step, args.warmup)
        step_ms = timed_ms(step, args.steps)
        write_ms = []
        for e in range(1, args.writes + 1):
            t0 = time.perf_counter()
            L._save_train_state(e, L.reader.state())
            write_ms.append(1e3 * (time.perf_counter() - t0))
        size = os.path.getsize(os.path.join(ck, 'train_state-%d.pt' % args.writes))
        steps = math.ceil(FLAGS['num_samples_train'].default / L.config.batch_size)
        w = statistics.median(write_ms)
        print(json.dumps({'case': name, 'batch': L.config.batch_size, 'step_ms': round(step_ms, 3), 'epoch_steps': steps,
                          'epoch_s': round(steps * step_ms / 1e3, 2), 'state_MB': round(size / 1e6, 1),
                          'write_ms': [round(v, 1) for v in write_ms], 'write_ms_median': round(w, 1),
                          'share_of_epoch': round(w / (steps * step_ms), 5)}))
        L.graph.graphs.clear()
    finally:
        shutil.rmtree(ck, ignore_errors=True)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=40)
    ap.add_argument('--warmup', type=int, default=8)
    ap.add_argument('--writes', type=int, default=3)
    args = ap.parse_args()
    print('card: %s' % card())
    measure('cis', cis, args)
    measure('flow', flow, args)


if __name__ == '__main__':
    main()
