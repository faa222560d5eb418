"""Training CLI with the reference's flag surface (its train.py:16-43): fixed seed 8964, flag dump, then
`AdversarialLearner().train(FLAGS)`.  Under torchrun every rank runs this file; only rank 0 prints.  --flow_dir (flow_flags.py)
trains on supplied flow instead of PWC-Net's; --flow_ckpt is then not read.  --ema_decay (ema_flags.py) keeps a moving average of the
generator and the recover net, which the validation IoU and model.best use.  --resumable (resume_flags.py) writes the full
training state every epoch and continues an interrupted run from it."""
import os
import pprint
import random
import sys

import numpy as np
import torch
from absl import flags as absl_flags

from unsupervised_detection_b200 import ema_flags, flow_flags, resume_flags
from unsupervised_detection_b200.common_flags import FLAGS, FLAG_NAMES
from unsupervised_detection_b200.models.adversarial_learner import AdversarialLearner

SEED = 8964


def seed_everything(seed=SEED):
    for fn in (torch.manual_seed, np.random.seed, random.seed):
        fn(seed)


def run(config):
    seed_everything()
    if int(os.environ.get('RANK', '0')) == 0:
        pprint.pprint({name: getattr(config, name) for name in FLAG_NAMES + ['flow_dir', 'ema_decay', 'resumable']})
    if config.checkpoint_dir:
        os.makedirs(config.checkpoint_dir, exist_ok=True)
    AdversarialLearner().train(config)


def main(argv):
    try:
        FLAGS(argv)
        flow_flags.check(FLAGS)
        ema_flags.check(FLAGS)
        resume_flags.check(FLAGS)
    except absl_flags.Error as err:
        sys.exit('%s\nUsage: %s ARGS\n%s' % (err, argv[0], FLAGS))
    try:
        run(FLAGS)
    except resume_flags.StateMismatch as err:          # the training state in --checkpoint_dir belongs to another run
        sys.exit('%s\nUsage: %s ARGS\n%s' % (err, argv[0], FLAGS))


if __name__ == "__main__":
    main(sys.argv)
