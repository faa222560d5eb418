"""Trains or fine-tunes PWC-Net (scope pwcnet) on Flying Chairs with tfoptflow's multi-scale flow loss, or without ground truth on the
frame pairs of a video dataset with the unsupervised census + smoothness loss, both as defined in
unsupervised_detection_b200/flow_train_graph.py.  Same flags, seed and flag dump as pretrain_recover.py, plus --flow_loss
(multiscale | robust | unsupervised), --smooth_weight (lambda_s of the unsupervised loss), --learning_rate, --lr_boundaries (steps after
which the rate halves), --weight_decay (L2 on the conv kernels) and --validate (every epoch: the end-point error on Flying Chairs' val split,
or the mean unsupervised objective over a video dataset's val pairs; pwcnet-best on improvement).  --flow_ckpt, when given, is the starting
point (fine-tuning); otherwise training starts from params_init.init_pwcnet.  The network input is img_height x img_width (multiples of
64, at least 128).

multiscale / robust need --dataset=FLYINGCHAIRS.  unsupervised also takes DAVIS2016, FBMS and SEGTRACK, whose training pairs come from
--train_partition with --train_crop and the temporal-shift flags, as in train.py; on Flying Chairs its ground truth is only used by
--validate.

It writes <checkpoint_dir>/pwcnet-<epoch> (TF V2 bundle of the pwcnet/* variables + .pt), which `--flow_ckpt` of train.py,
test_generator*.py, pretrain_recover.py and export_flow.py read.  Under torchrun every rank runs this file; only rank 0 prints."""
import os
import pprint
import sys

from absl import flags as absl_flags

from train import seed_everything
from unsupervised_detection_b200 import flow_flags
from unsupervised_detection_b200.common_flags import FLAGS, FLAG_NAMES, define_validate

TRAIN_FLOW_FLAGS = ['flow_loss', 'smooth_weight', 'learning_rate', 'lr_boundaries', 'weight_decay', 'validate']
UNSUP_DATASETS = ('FLYINGCHAIRS', 'DAVIS2016', 'FBMS', 'SEGTRACK')
if 'flow_loss' not in FLAGS:
    absl_flags.DEFINE_enum('flow_loss', 'multiscale', ['multiscale', 'robust', 'unsupervised'], "flow loss: 'multiscale' = ||d||_2 to "
                           "the ground truth (pretraining), 'robust' = (|d0| + |d1| + 0.01)^0.4 (fine-tuning), 'unsupervised' = "
                           "occlusion-masked census + smoothness on frame pairs without ground truth (fine-tuning on the target videos)")
    absl_flags.DEFINE_float('smooth_weight', 3.0, 'lambda_s: weight of the second-order smoothness term of the unsupervised loss')
    absl_flags.DEFINE_float('learning_rate', 1e-4, 'Adam learning rate of the first step')
    absl_flags.DEFINE_list('lr_boundaries', [], 'steps after which the learning rate halves (comma-separated, increasing)')
    absl_flags.DEFINE_float('weight_decay', 4e-4, 'L2 weight decay gamma of the conv kernels (loss term gamma/2 ||w||^2; biases are not decayed)')
define_validate()


def lr_boundaries(config):
    """--lr_boundaries as increasing positive ints; IllegalFlagValueError otherwise."""
    try:
        b = [int(v) for v in config.lr_boundaries]
    except ValueError:
        raise absl_flags.IllegalFlagValueError('--lr_boundaries must be step numbers, got %r' % (config.lr_boundaries,))
    if any(v < 1 for v in b) or b != sorted(set(b)):
        raise absl_flags.IllegalFlagValueError('--lr_boundaries must be increasing positive steps, got %r' % (b,))
    return b


def check_flags(config):
    """Usage errors of train_flow.py -> absl_flags.IllegalFlagValueError."""
    from unsupervised_detection_b200.flow_train_graph import check_size
    unsup = config.flow_loss == 'unsupervised'
    if unsup and config.dataset not in UNSUP_DATASETS:
        raise absl_flags.IllegalFlagValueError('--flow_loss=unsupervised trains on --dataset in %s, not %s'
                                               % (' / '.join(UNSUP_DATASETS), config.dataset))
    if not unsup and config.dataset != 'FLYINGCHAIRS':
        raise absl_flags.IllegalFlagValueError('train_flow.py trains on Flying Chairs: --dataset=FLYINGCHAIRS, not %s' % config.dataset)
    if unsup and config.flow_dir:
        raise absl_flags.IllegalFlagValueError('--flow_dir replaces PWC-Net, which --flow_loss=unsupervised trains: drop one of them')
    if not config.smooth_weight >= 0:
        raise absl_flags.IllegalFlagValueError('--smooth_weight must be >= 0')
    if not config.checkpoint_dir:
        raise absl_flags.IllegalFlagValueError('--checkpoint_dir is needed: the pwcnet-<epoch> checkpoints are written there')
    try:
        check_size(config.img_height, config.img_width)
    except ValueError as err:
        raise absl_flags.IllegalFlagValueError('--img_height / --img_width: %s' % err)
    flow_flags.check(config)
    if not config.learning_rate > 0 or config.weight_decay < 0:
        raise absl_flags.IllegalFlagValueError('--learning_rate must be > 0 and --weight_decay >= 0')
    lr_boundaries(config)
    if config.validate and config.dataset == 'FLYINGCHAIRS':
        from unsupervised_detection_b200.data.flyingchairs_data_utils import SPLIT_FILE
        if not os.path.isfile(os.path.join(config.root_dir, SPLIT_FILE)):
            raise absl_flags.IllegalFlagValueError('--validate needs a val split: %s in --root_dir' % SPLIT_FILE)
    elif config.validate and not val_pairs(config):
        raise absl_flags.IllegalFlagValueError('--validate needs val pairs: --dataset=%s has none in --root_dir' % config.dataset)


def val_pairs(config):
    """The number of frame pairs of the val partition of a video dataset (0 when the reader finds none)."""
    from export_flow import make_reader
    try:
        return len(make_reader(config).test_frame_pairs('val', config.test_temporal_shift))
    except (IOError, OSError, AssertionError):
        return 0


def run(config):
    from unsupervised_detection_b200.models.flow_learner import FlowLearner
    seed_everything()
    if int(os.environ.get('RANK', '0')) == 0:
        pprint.pprint({name: getattr(config, name) for name in FLAG_NAMES + TRAIN_FLOW_FLAGS})
    os.makedirs(config.checkpoint_dir, exist_ok=True)
    FlowLearner().train_flow(config)


def main(argv):
    try:
        FLAGS(argv)
        check_flags(FLAGS)
    except absl_flags.Error as err:
        sys.exit('%s\nUsage: %s ARGS\n%s' % (err, argv[0], FLAGS))
    run(FLAGS)


if __name__ == "__main__":
    main(sys.argv)
