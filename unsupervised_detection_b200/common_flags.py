"""The reference's config system (common_flags.py:5-55) on absl.flags (API-compatible successor of python-gflags):
the same 31 flag names, types and defaults, declared from one table; the whole FLAGS object is passed around as `config`."""
from absl import flags as gflags

FLAGS = gflags.FLAGS


# (kind, name, default, what it controls) -- names, types and defaults are the reference's command-line surface
# (common_flags.py:5-55 of the reference); descriptions are this package's own.
_SPEC = [
    # ---- training
    ('integer', 'img_width', 384, 'network input width in pixels (frames are read at 384x640 and resized to this)'),
    ('integer', 'img_height', 192, 'network input height in pixels'),
    ('integer', 'batch_size', 16, 'frame pairs per step for the WHOLE job (sharded over the ranks under torchrun)'),
    ('float', 'beta1', 0.9, 'Adam first-moment decay'),
    ('float', 'flow_normalizer', 80.0, 'PWC-Net flow is divided by this constant before it enters the loss'),
    ('integer', 'max_epochs', 40, 'stop after this many epochs'),
    ('integer', 'num_samples_train', 5000, 'frame pairs that count as one epoch (independent of the dataset size)'),
    ('float', 'train_crop', 0.9, 'smallest random crop fraction used for training augmentation'),
    ('integer', 'max_temporal_len', 2, 'largest frame distance between the two images of a training pair'),
    ('integer', 'min_temporal_len', 1, 'smallest frame distance between the two images of a training pair'),
    ('float', 'cbn', 0.5, 'Charbonnier exponent: 0.5 behaves like L1, 1.0 like L2'),
    ('float', 'epsilon', 75.0, 'added to the denominators of the reduction rates'),
    ('integer', 'iters_rec', 1, 'recover (inpainter) updates per cycle; raise it when the recover net starts from scratch'),
    ('integer', 'iters_gen', 3, 'generator (mask) updates per cycle'),
    ('integer', 'num_threads', 6, 'host threads decoding and augmenting frames'),
    ('bool', 'resume_train', False, 'continue from full_model_ckpt or the newest checkpoint in checkpoint_dir'),
    # ---- paths
    ('string', 'root_dir', '/your/path/to/DAVIS_2016', 'dataset root folder'),
    ('string', 'train_partition', 'trainval', 'partition used for training: train / val / trainval'),
    ('string', 'dataset', 'DAVIS2016', 'DAVIS2016, FBMS, SEGTRACK, or SYNTHETIC (seeded synthetic frame pairs); pretrain_recover.py '
                                       'also reads FLYINGCHAIRS'),
    ('string', 'recover_ckpt', '', 'pre-trained recover net (TF checkpoint prefix or .pt); empty = train it from scratch'),
    ('string', 'flow_ckpt', '', 'pre-trained PWC-Net (mandatory; TF checkpoint prefix, its .index/.data file, or .pt)'),
    ('string', 'full_model_ckpt', '', 'checkpoint of all networks, used together with resume_train'),
    ('string', 'checkpoint_dir', '', 'experiment folder: checkpoints and TensorBoard event files go here'),
    # ---- logging
    ('integer', 'summary_freq', 30, 'write TensorBoard summaries and print the losses every this many iterations'),
    ('integer', 'save_freq', 5, 'save model-<epoch> every this many epochs (model.best is saved on every improvement)'),
    # ---- evaluation
    ('bool', 'generate_visualization', False, 'dump PNG overlays and .mat files while evaluating'),
    ('float', 'test_crop', 0.9, 'central crop fraction applied to evaluation frames'),
    ('integer', 'test_temporal_shift', 1, 'frame distance between the two evaluation images (negative looks backwards)'),
    ('string', 'ckpt_file', '', 'checkpoint evaluated by test_generator*.py'),
    ('string', 'test_partition', 'val', 'partition evaluated: train / val / trainval'),
    ('string', 'test_save_dir', '', 'output folder of the evaluation dumps'),
]
FLAG_NAMES = [name for _, name, _, _ in _SPEC]


def _define():
    if 'img_width' in FLAGS:
        return
    for kind, name, default, text in _SPEC:
        getattr(gflags, 'DEFINE_' + kind)(name, default, text)


_define()


def define_validate():
    """--validate, shared by pretrain_recover.py and train_flow.py (not one of the reference's flags, so not in FLAG_NAMES): defined once,
    with one help text, by whichever of the two scripts is imported first."""
    if 'validate' not in FLAGS:
        gflags.DEFINE_bool('validate', False, 'score the held-out end-point error on the val split at every epoch end and save the '
                                              'best checkpoint (recover-best / pwcnet-best) when it improves; needs --dataset=FLYINGCHAIRS '
                                              'with its split file, or for train_flow.py --flow_loss=unsupervised a mask dataset '
                                              'with val pairs (scored by the unsupervised objective)')


class Config(object):
    """Plain-attribute stand-in for the parsed FLAGS object (handy for tests / bench): same names and defaults."""

    def __init__(self, **kw):
        for n in FLAG_NAMES:
            setattr(self, n, FLAGS[n].default)
        for k, v in kw.items():
            if k not in FLAG_NAMES:
                raise AttributeError('unknown flag ' + k)
            setattr(self, k, v)
