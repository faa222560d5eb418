"""--resumable: continue an interrupted training run exactly where its last completed epoch ended.  It is not one of the reference's flags,
so it is defined here once and common_flags.py keeps the reference's flag surface.  The learner (models/adversarial_learner.py) imports
this module, so train.py, pretrain_recover.py and train_flow.py accept it, as they do --ema_decay (ema_flags.py).

With --resumable every epoch end writes <checkpoint_dir>/train_state-<epoch>.pt (train_state.py): the live weights, Adam's moments, the
moving averages, the device step counter, the learner's counters and every rank's reader position.  A run started with the flag continues
from the newest such file when checkpoint_dir holds one, and starts afresh otherwise, so one command line both starts a run and continues
it after an interruption.  --resume_train (the reference's restart from a checkpoint's weights) is a different starting state and cannot
be combined with it."""
from absl import flags as gflags

from .common_flags import FLAGS

if 'resumable' not in FLAGS:
    gflags.DEFINE_bool('resumable', False, 'write the full training state (weights, Adam moments, averages, step counters, reader '
                                           'positions) to <checkpoint_dir>/train_state-<epoch>.pt at every epoch end, and continue from the '
                                           'newest one when it exists; the continued run is bit-identical to an uninterrupted one')


class StateMismatch(gflags.IllegalFlagValueError):
    """A training state file that does not belong to this run's command line: a usage error."""


def check(config):
    """--resumable's usage errors -> gflags.IllegalFlagValueError: it needs --checkpoint_dir and excludes --resume_train."""
    if not getattr(config, 'resumable', False):
        return
    if not config.checkpoint_dir:
        raise gflags.IllegalFlagValueError('--resumable needs --checkpoint_dir: the training state is written there')
    if config.resume_train:
        raise gflags.IllegalFlagValueError('--resumable and --resume_train both give the starting state: drop one of them')
