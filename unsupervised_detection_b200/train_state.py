"""The training state file of --resumable (resume_flags.py): <checkpoint_dir>/train_state-<epoch>.pt, a torch.save dict written by rank 0
at the end of epoch <epoch>, after that epoch's checkpoints and validation, so a state for epoch e means every output of epoch e is on disk.

    format        FORMAT
    kind          'adversarial' (train.py) | 'pretrain_recover' | 'flow' (train_flow.py)
    epoch         the epoch it ends
    world         the number of ranks
    flags         trajectory(config): every flag the trajectory depends on
    frozen_crc    CRC-32C of the frozen PWC-Net parameters the run reads, None when it reads none
    global_step, step, min_val_iou, min_val_epe     the learner's counters
    stores        {scope: {'flat', 'm', 'v'[, 'shadow']: fp32 CPU tensors}} of every trained ParamStore
    step_state    the graph's int64 device step counter
    readers       per rank: {'train': the training reader's position at the next batch to train on, 'train_now': its position after
                  everything the run has drawn, 'val': train.py's validation reader's position, or None}

A file is written as <name>.tmp and renamed, so a file under its final name is complete; a .tmp left by an interrupted write is ignored
and removed by the next write.  Only the newest KEEP files stay."""
import os
import re

import torch

from .resume_flags import StateMismatch

FORMAT = 1
KEEP = 2
KINDS = {'adversarial': 'train.py', 'pretrain_recover': 'pretrain_recover.py', 'flow': 'train_flow.py'}
_NAME = re.compile(r'^train_state-(\d+)\.pt$')

# Flags that change what a run computes.  The others (max_epochs, root_dir, num_threads, summary_freq, save_freq, ...) may differ when
# a run is continued.
TRAJECTORY_FLAGS = ('img_height', 'img_width', 'batch_size', 'num_samples_train', 'dataset', 'train_partition', 'train_crop', 'test_crop',
                    'max_temporal_len', 'min_temporal_len', 'test_temporal_shift', 'iters_rec', 'iters_gen', 'cbn', 'epsilon', 'beta1',
                    'flow_normalizer', 'ema_decay', 'flow_loss', 'flow_aug', 'learning_rate', 'lr_boundaries', 'weight_decay',
                    'smooth_weight', 'box_min', 'box_max', 'pretrain_flow')


def trajectory(config):
    """{flag: value} of TRAJECTORY_FLAGS (None for a flag the script does not define), whether --flow_dir is set, and PWC-Net's option
    set."""
    from .models.PWCNet import model_pwcnet
    out = {n: getattr(config, n, None) for n in TRAJECTORY_FLAGS}
    if out['lr_boundaries'] is not None:
        out['lr_boundaries'] = [int(b) for b in out['lr_boundaries']]
    out['flow_dir'] = bool(getattr(config, 'flow_dir', ''))
    out['pwc_options'] = repr(sorted((k, v) for k, v in model_pwcnet._DEFAULT_PWCNET_TEST_OPTIONS.items() if k not in ('verbose', 'ckpt_path')))
    return out


def path(checkpoint_dir, epoch):
    return os.path.join(checkpoint_dir, 'train_state-%d.pt' % epoch)


def epochs(checkpoint_dir):
    """The epochs of the complete state files in checkpoint_dir, ascending."""
    if not os.path.isdir(checkpoint_dir):
        return []
    return sorted(int(m.group(1)) for m in map(_NAME.match, os.listdir(checkpoint_dir)) if m)


def newest(checkpoint_dir):
    """The state file of the latest epoch in checkpoint_dir, or None."""
    e = epochs(checkpoint_dir)
    return path(checkpoint_dir, e[-1]) if e else None


def write(checkpoint_dir, state):
    """Writes `state` as the file of epoch state['epoch'], atomically, and keeps the newest KEEP files -> its path."""
    for f in os.listdir(checkpoint_dir):
        if f.startswith('train_state-') and f.endswith('.pt.tmp'):
            os.remove(os.path.join(checkpoint_dir, f))
    out = path(checkpoint_dir, state['epoch'])
    with open(out + '.tmp', 'wb') as f:
        torch.save(state, f)
        f.flush()
        os.fsync(f.fileno())
    os.replace(out + '.tmp', out)
    for e in epochs(checkpoint_dir)[:-KEEP]:
        os.remove(path(checkpoint_dir, e))
    return out


def load(file):
    """The state dict of `file` (CPU tensors); StateMismatch for a file of another format."""
    st = torch.load(file, map_location='cpu', weights_only=True)
    if st.get('format') != FORMAT:
        raise StateMismatch('--resumable: %s has format %r, this version reads %d' % (file, st.get('format'), FORMAT))
    return st


def check(state, file, kind, world, flags, frozen_crc):
    """StateMismatch naming the flag and both values when `state` (read from `file`) was written by another script, on another number of
    ranks, with another trajectory flag or from other frozen PWC-Net parameters than this run's."""
    if state['kind'] != kind:
        raise StateMismatch('--resumable: %s was written by %s, not %s' % (file, KINDS[state['kind']], KINDS[kind]))
    if state['world'] != world:
        raise StateMismatch('--resumable: %s was written by %d ranks, this run has %d' % (file, state['world'], world))
    for name, v in flags.items():
        if state['flags'].get(name) != v:
            raise StateMismatch('--resumable: %s was written with --%s=%r, this run has --%s=%r'
                                % (file, name, state['flags'].get(name), name, v))
    if state['frozen_crc'] != frozen_crc:
        raise StateMismatch('--resumable: %s was written with other PWC-Net parameters (CRC-32C %s), this run reads --flow_ckpt with %s'
                            % (file, state['frozen_crc'], frozen_crc))
