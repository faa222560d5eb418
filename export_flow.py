"""Writes PWC-Net's optical flow of every frame pair a dataset reader can draw into a --flow_dir tree, so that train.py,
test_generator.py, test_generator_ensemble.py and pretrain_recover.py can later run on it with --flow_dir and no PWC-Net in the loop.

The pairs are the reader's own lists (Davis2016Reader.frame_pairs) for --train_partition, 'val' (the validation pass of train.py) and
--test_partition: every training pair at every shift in [--min_temporal_len, --max_temporal_len] in both directions, and the test pairs
at --test_temporal_shift.  Frames are read unaugmented and uncropped at 384x640, PWC-Net (--flow_ckpt) runs on them in batches of
--batch_size, and each pair's field is written as one Middlebury .flo file at 384x640, (u, v) = (-flow1, -flow0), the exact inverse
of the readers' pwc_flow_from_uv, under the name data/davis2016_data_utils.flow_file gives it.  Under torchrun, rank r writes pairs
r, r + world, ...: the ranks write disjoint files.  --use_ema (ema_flags.py) runs the moving average of a pwcnet-<epoch> written by
train_flow.py --ema_decay."""
import os
import sys
from concurrent.futures import ThreadPoolExecutor

from absl import flags as absl_flags

from unsupervised_detection_b200 import ema_flags, flow_flags  # noqa: F401  (ema_flags defines --use_ema)
from unsupervised_detection_b200.common_flags import FLAGS


def check_flags(config):
    """Usage errors -> absl_flags.IllegalFlagValueError."""
    if not config.flow_dir:
        raise absl_flags.IllegalFlagValueError('--flow_dir is needed: the .flo files are written there')
    flow_flags.check(config, must_exist=False)
    if not config.flow_ckpt:
        raise absl_flags.IllegalFlagValueError('--flow_ckpt is needed: the exported flow is PWC-Net\'s')


def make_reader(config):
    """The dataset reader of --dataset on --root_dir (frames only: no flow_dir)."""
    from unsupervised_detection_b200.data.davis2016_data_utils import Davis2016Reader
    from unsupervised_detection_b200.data.fbms_data_utils import FBMS59Reader
    from unsupervised_detection_b200.data.segtrackv2_data_utils import SegTrackV2Reader
    cls = {'DAVIS2016': Davis2016Reader, 'FBMS': FBMS59Reader, 'SEGTRACK': SegTrackV2Reader}[config.dataset]
    return cls(config.root_dir, max_temporal_len=config.max_temporal_len, min_temporal_len=config.min_temporal_len,
               num_threads=config.num_threads)


def export_pairs(config, rd):
    """Sorted, without repeats: the frame pairs of --train_partition, 'val' and --test_partition (see the module docstring)."""
    parts = []
    for p in (config.train_partition, 'val', config.test_partition):
        if p not in parts:
            parts.append(p)
    return sorted(set(pr for p in parts for pr in rd.frame_pairs(p, config.test_temporal_shift)))


def export(config):
    """-> the number of .flo files this rank wrote."""
    import numpy as np
    import torch
    from unsupervised_detection_b200.data.davis2016_data_utils import Davis2016Reader, flow_file
    from unsupervised_detection_b200.data.flyingchairs_data_utils import uv_from_pwc_flow, write_flo
    from unsupervised_detection_b200 import params_init
    from unsupervised_detection_b200.models.PWCNet import model_pwcnet
    from unsupervised_detection_b200.models.adversarial_learner import AdversarialLearner
    from unsupervised_detection_b200.step_graph import CISGraph
    L = AdversarialLearner()
    L.config = config
    L._init_dist()
    rank, world, B = L.rank, L.world, config.batch_size
    pairs = export_pairs(config, make_reader(config))
    mine = pairs[rank::world]
    if rank == 0:
        print('Exporting the flow of {} frame pairs to {} ({} rank(s))'.format(len(pairs), config.flow_dir, world))
    L.graph = g = CISGraph(config.img_height, config.img_width, B, device=L.device, with_pwc=True, train=False,
                           pwc_options=model_pwcnet._DEFAULT_PWCNET_TEST_OPTIONS)
    # the graph also holds the generator and the recover net, which forward_flow never runs: any values do
    g.load_params(dict(params_init.init_generator(), **params_init.init_recover(), **L.flow_net_params()))
    pool = ThreadPoolExecutor(max_workers=max(1, config.num_threads))
    for k in range(0, len(mine), B):
        chunk = mine[k:k + B]
        padded = chunk + [chunk[-1]] * (B - len(chunk))          # a short last batch repeats its last pair; only real pairs are written
        frames = list(pool.map(Davis2016Reader.preprocess_image, [f for pr in padded for f in pr]))
        g.feed(torch.from_numpy(np.stack(frames[0::2])), torch.from_numpy(np.stack(frames[1::2])))
        g.forward_flow()
        flow = g.flow_full.cpu().numpy()
        for j, (f1, f2) in enumerate(chunk):
            write_flo(flow_file(config.flow_dir, config.root_dir, f1, f2), uv_from_pwc_flow(flow[j]))
    pool.shutdown()
    d = torch.distributed
    if world > 1 and d.is_initialized():
        d.barrier()
    if rank == 0:
        print('Success: wrote the flow of {} frame pairs'.format(len(pairs)))
    return len(mine)


def main(argv):
    try:
        FLAGS(argv)
        check_flags(FLAGS)
    except absl_flags.Error as err:
        sys.exit('%s\nUsage: %s ARGS\n%s' % (err, argv[0], FLAGS))
    os.makedirs(FLAGS.flow_dir, exist_ok=True)
    export(FLAGS)


if __name__ == "__main__":
    main(sys.argv)
