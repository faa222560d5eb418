"""Pretrains the recover network (the flow inpainter, scope FlownetS) on box-shaped flow occlusions: the recover step of train.py with one
random box per sample in place of the generator's mask.  Same flags, seed and flag dump as train.py, plus --box_min / --box_max (box side
range as fractions of each image side), --pretrain_flow (PWC-Net's flow, or the dataset's ground-truth flow: Flying Chairs' own, or the
supplied flow of a mask dataset under --flow_dir), --validate (held-out EPE
every epoch, recover-best on improvement) and --ema_decay (a moving average of the recover net's weights, which the validation and
recover-best use) and --resumable (continue an interrupted run from its last epoch).  It writes <checkpoint_dir>/recover-<epoch> (TF V2 bundle + .pt), which
`train.py --recover_ckpt=<checkpoint_dir>/recover-<epoch>` then starts adversarial training from.  Under torchrun every rank runs this
file; only rank 0 prints."""
import os
import pprint
import sys

from absl import flags as absl_flags

from train import seed_everything
from unsupervised_detection_b200 import ema_flags, flow_flags, resume_flags
from unsupervised_detection_b200.common_flags import FLAGS, FLAG_NAMES, define_validate
from unsupervised_detection_b200.step_graph import box_sides

PRETRAIN_FLAGS = ['box_min', 'box_max', 'pretrain_flow', 'validate', 'flow_dir', 'ema_decay', 'resumable']
if 'box_min' not in FLAGS:
    absl_flags.DEFINE_float('box_min', 0.1, 'smallest box side, as a fraction of the image side (per axis)')
    absl_flags.DEFINE_float('box_max', 0.5, 'largest box side, as a fraction of the image side (per axis)')
    absl_flags.DEFINE_enum('pretrain_flow', 'pwc', ['pwc', 'gt'], "flow the recover net learns to inpaint: 'pwc' = PWC-Net's flow of "
                           "the frame pair (needs --flow_ckpt), 'gt' = the dataset's ground-truth flow (FLYINGCHAIRS, or DAVIS2016 / FBMS / "
                           "SEGTRACK with --flow_dir)")
define_validate()


def check_flags(config):
    """Usage errors of the pretraining flags -> absl_flags.IllegalFlagValueError."""
    from unsupervised_detection_b200.models.adversarial_learner import FLOW_DATASETS, MASK_DATASETS, has_flow
    try:
        box_sides(config.box_min, config.box_max, config.img_height, config.img_width)
    except ValueError as err:
        raise absl_flags.IllegalFlagValueError(str(err))
    if not config.checkpoint_dir:
        raise absl_flags.IllegalFlagValueError('--checkpoint_dir is needed: the recover-<epoch> checkpoints are written there')
    flow_flags.check(config)
    ema_flags.check(config)
    resume_flags.check(config)
    if config.pretrain_flow == 'gt' and not has_flow(config.dataset, config.flow_dir):
        raise absl_flags.IllegalFlagValueError('--pretrain_flow=gt needs a dataset with ground-truth flow (%s) or --flow_dir with %s, not %s'
                                               % (', '.join(FLOW_DATASETS), ' / '.join(MASK_DATASETS), config.dataset))
    if config.flow_dir and config.pretrain_flow != 'gt':
        raise absl_flags.IllegalFlagValueError('--flow_dir replaces PWC-Net: it needs --pretrain_flow=gt')
    if config.validate:
        from unsupervised_detection_b200.data.flyingchairs_data_utils import SPLIT_FILE
        if config.dataset != 'FLYINGCHAIRS' or not os.path.isfile(os.path.join(config.root_dir, SPLIT_FILE)):
            raise absl_flags.IllegalFlagValueError('--validate needs a val split: --dataset=FLYINGCHAIRS with %s in --root_dir'
                                                   % SPLIT_FILE)


def run(config):
    from unsupervised_detection_b200.models.adversarial_learner import AdversarialLearner
    seed_everything()
    if int(os.environ.get('RANK', '0')) == 0:
        pprint.pprint({name: getattr(config, name) for name in FLAG_NAMES + PRETRAIN_FLAGS})
    if config.checkpoint_dir:
        os.makedirs(config.checkpoint_dir, exist_ok=True)
    AdversarialLearner().pretrain_recover(config)


def main(argv):
    try:
        FLAGS(argv)
        check_flags(FLAGS)
    except absl_flags.Error as err:
        sys.exit('%s\nUsage: %s ARGS\n%s' % (err, argv[0], FLAGS))
    try:
        run(FLAGS)
    except resume_flags.StateMismatch as err:          # the training state in --checkpoint_dir belongs to another run
        sys.exit('%s\nUsage: %s ARGS\n%s' % (err, argv[0], FLAGS))


if __name__ == "__main__":
    main(sys.argv)
