"""--flow_dir, the script-level flag of train.py, test_generator.py, test_generator_ensemble.py, pretrain_recover.py and export_flow.py.
It is not one of the reference's flags, so it is defined here once and common_flags.py keeps the reference's flag surface.  The
learner (models/adversarial_learner.py) imports this module, so every script that drives it accepts the flag, and it checks the value
(validate) when it opens a dataset.

--flow_dir=<dir>: read the flow of every frame pair from the .flo files under <dir> (data/davis2016_data_utils.flow_file names them;
export_flow.py writes them) in place of running PWC-Net.  '' (the default) keeps PWC-Net in the loop."""
import os

from absl import flags as gflags

from .common_flags import FLAGS

if 'flow_dir' not in FLAGS:
    gflags.DEFINE_string('flow_dir', '', "directory of supplied optical flow (.flo per frame pair, see export_flow.py) used in place of "
                                         "PWC-Net's flow; DAVIS2016 / FBMS / SEGTRACK only.  '' = run PWC-Net")


def validate(config, must_exist=True):
    """config.flow_dir (absent or '' = PWC-Net's flow) against config.dataset: ValueError for a dataset without frame-pair readers,
    IOError (must_exist) for a directory that does not exist."""
    from .models.adversarial_learner import MASK_DATASETS
    fd = getattr(config, 'flow_dir', '')
    if not fd:
        return
    if config.dataset not in MASK_DATASETS:
        raise ValueError('--flow_dir needs --dataset in %s, not %s' % (' / '.join(MASK_DATASETS), config.dataset))
    if must_exist and not os.path.isdir(fd):
        raise IOError('--flow_dir=%s is not a directory' % fd)


def check(config, must_exist=True):
    """validate() as a usage error of the command line: gflags.IllegalFlagValueError."""
    try:
        validate(config, must_exist)
    except (ValueError, IOError) as err:
        raise gflags.IllegalFlagValueError(str(err))
