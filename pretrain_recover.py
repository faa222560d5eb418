"""Pretrains the recover network (the flow inpainter, scope FlownetS) on box-shaped flow occlusions: the recover step of train.py with one
random box per sample in place of the generator's mask.  Same flags, seed and flag dump as train.py, plus --box_min / --box_max (box side
range as fractions of each image side).  It writes <checkpoint_dir>/recover-<epoch> (TF V2 bundle + .pt), which
`train.py --recover_ckpt=<checkpoint_dir>/recover-<epoch>` then starts adversarial training from.  Under torchrun every rank runs this
file; only rank 0 prints."""
import os
import pprint
import sys

from absl import flags as absl_flags

from train import seed_everything
from unsupervised_detection_b200.common_flags import FLAGS, FLAG_NAMES
from unsupervised_detection_b200.step_graph import box_sides

BOX_FLAGS = ['box_min', 'box_max']
if 'box_min' not in FLAGS:
    absl_flags.DEFINE_float('box_min', 0.1, 'smallest box side, as a fraction of the image side (per axis)')
    absl_flags.DEFINE_float('box_max', 0.5, 'largest box side, as a fraction of the image side (per axis)')


def run(config):
    from unsupervised_detection_b200.models.adversarial_learner import AdversarialLearner
    seed_everything()
    if int(os.environ.get('RANK', '0')) == 0:
        pprint.pprint({name: getattr(config, name) for name in FLAG_NAMES + BOX_FLAGS})
    if config.checkpoint_dir:
        os.makedirs(config.checkpoint_dir, exist_ok=True)
    AdversarialLearner().pretrain_recover(config)


def main(argv):
    try:
        FLAGS(argv)
        try:
            box_sides(FLAGS.box_min, FLAGS.box_max, FLAGS.img_height, FLAGS.img_width)
        except ValueError as err:
            raise absl_flags.IllegalFlagValueError(str(err))
        if not FLAGS.checkpoint_dir:
            raise absl_flags.IllegalFlagValueError('--checkpoint_dir is needed: the recover-<epoch> checkpoints are written there')
    except absl_flags.Error as err:
        sys.exit('%s\nUsage: %s ARGS\n%s' % (err, argv[0], FLAGS))
    run(FLAGS)


if __name__ == "__main__":
    main(sys.argv)
