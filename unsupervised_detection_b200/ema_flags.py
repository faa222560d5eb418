"""--ema_decay and --use_ema: the moving average of the trained weights, tf.train.ExponentialMovingAverage's semantics and names.  They
are not among the reference's flags, so they are defined here once and common_flags.py keeps the reference's flag surface.  The learner
(models/adversarial_learner.py) imports this module, so every script that drives it accepts both, as with --flow_dir (flow_flags.py).

--ema_decay=<d> (train.py, pretrain_recover.py, train_flow.py): 0 (the default) keeps no average; 0 < d < 1 keeps
shadow = shadow - (shadow - w) * (1 - min(d, (1 + t) / (10 + t))) of every trained variable after each optimiser step t, on the GPU.
Epoch checkpoints then also hold <var>/ExponentialMovingAverage, the validation scores the averages and the best checkpoint holds them
under the plain names.

--use_ema: read <var>/ExponentialMovingAverage in place of <var> from the checkpoint of --ckpt_file (test_generator.py,
test_generator_ensemble.py: the generator, and the recover net where it has averages) and of --flow_ckpt (PWC-Net: export_flow.py, and
every other script that reads --flow_ckpt)."""
from absl import flags as gflags

from .common_flags import FLAGS
from .engine import check_ema_decay

if 'ema_decay' not in FLAGS:
    gflags.DEFINE_float('ema_decay', 0.0, 'decay of the exponential moving average of the trained weights (0 < d < 1, e.g. 0.999); the '
                                          'averages go into every checkpoint as <var>/ExponentialMovingAverage, and the validation and '
                                          'the best checkpoint use them.  0 = no average')
    gflags.DEFINE_bool('use_ema', False, 'read the moving averages <var>/ExponentialMovingAverage of the trained networks from --ckpt_file '
                                         'and --flow_ckpt in place of the variables (a checkpoint written with --ema_decay)')


def check(config):
    """config.ema_decay (absent = 0) as a usage error of the command line: gflags.IllegalFlagValueError unless 0 or in (0, 1)."""
    try:
        check_ema_decay(getattr(config, 'ema_decay', 0.0))
    except ValueError as err:
        raise gflags.IllegalFlagValueError('--' + str(err))
