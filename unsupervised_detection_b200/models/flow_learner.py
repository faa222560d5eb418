"""FlowLearner: trains or fine-tunes PWC-Net (scope pwcnet) on Flying Chairs with the multi-scale flow loss, or on the frame pairs of
DAVIS2016 / FBMS / SEGTRACK (or Flying Chairs) with the unsupervised loss (flow_train_graph.py), and writes pwcnet-<epoch> checkpoints
that --flow_ckpt of train.py, test_generator*.py, pretrain_recover.py and export_flow.py read.

It is AdversarialLearner's counterpart for the flow network: the same process setup (one process per GPU under torchrun, the global
batch sharded over ranks, one NCCL all-reduce of the flat gradient per step), reader, summaries and checkpoint writer.  The PWC-Net option
set is model_pwcnet._DEFAULT_PWCNET_TEST_OPTIONS, as for every other graph.
"""
import math
import time
from itertools import count

import torch

from .adversarial_learner import AdversarialLearner, FLOW_DATASETS, MASK_DATASETS, _dist
from .PWCNet import model_pwcnet
from .. import params_init
from ..flow_train_graph import FlowTrainGraph
from ..step_graph import PWC_H, PWC_W


# the scalars train_flow writes every summary_freq steps, in this order
SUMMARY_KEYS = {'multiscale': ['flow_loss'] + ['flow_loss_l%d' % l for l in (6, 5, 4, 3, 2)],
                'unsupervised': ['flow_loss', 'flow_loss_photo', 'flow_loss_smooth']}
SUMMARY_KEYS['robust'] = SUMMARY_KEYS['multiscale']


def learning_rate_at(step, base, boundaries):
    """Rate of update number `step` (1-based): `base`, halved once for every boundary b < step (updates after the first b run at half
    the rate)."""
    return base * 0.5 ** sum(1 for b in boundaries if step > b)


class FlowLearner(AdversarialLearner):
    _lr = None                                          # the rate last written to the graph
    min_val_epe = math.inf

    def build_flow_graph(self):
        """FlowTrainGraph at img_height x img_width on the 384x640 batches (the frames are resized on the device; the supervised losses
        sample their targets from the 384x640 flow); parameters from --flow_ckpt when given, else params_init.init_pwcnet.  The
        unsupervised loss also reads the training pairs of a mask dataset (--train_partition, --train_crop, the temporal shifts)."""
        cfg = self.config
        loss = getattr(cfg, 'flow_loss', 'multiscale')
        ok = FLOW_DATASETS + (MASK_DATASETS if loss == 'unsupervised' else ())
        if cfg.dataset not in ok:
            raise IOError('PWC-Net training with the %s loss needs a dataset in %s, got %s' % (loss, ', '.join(ok), cfg.dataset))
        self._init_dist()
        if cfg.batch_size % self.world:
            raise ValueError('batch_size must be divisible by the number of ranks')
        self.local_batch = cfg.batch_size // self.world
        self._pretrain = True                           # load_training_data: Flying Chairs' train pairs
        self.load_training_data()
        self.graph = FlowTrainGraph(cfg.img_height, cfg.img_width, self.local_batch, options=model_pwcnet._DEFAULT_PWCNET_TEST_OPTIONS,
                                    global_batch=cfg.batch_size, device=self.device, in_hw=(PWC_H, PWC_W),
                                    loss=loss, weight_decay=getattr(cfg, 'weight_decay', 4e-4),
                                    lr=self._rate(1), beta1=cfg.beta1, smooth_weight=getattr(cfg, 'smooth_weight', 3.0))
        self._lr = self._rate(1)
        self.train_steps_per_epoch = int(math.ceil(cfg.num_samples_train / cfg.batch_size))
        names = [e[0] for e in self.graph.store.entries]
        fc = getattr(cfg, 'flow_ckpt', '')
        if fc and not fc.startswith('synthetic'):
            if not self._is_ckpt(fc):
                raise IOError("Could not find flow ckpt file. Aborting.")
            p = self._read_ckpt(fc, names)[0]
            print("Flow net loaded from {}".format(fc))
        else:
            p = params_init.init_pwcnet(self.graph.store.entries)
        self.graph.load_params(p)

    def _rate(self, step):
        cfg = self.config
        return learning_rate_at(step, getattr(cfg, 'learning_rate', 1e-4), [int(b) for b in getattr(cfg, 'lr_boundaries', None) or ()])

    def _flow_batch(self, batch):
        """(img1, img2, ground-truth flow) of a Flying Chairs batch (img1, img2, flow, names); (img1, img2, None) of a mask dataset's
        (img1, img2, seg1, names): no ground truth."""
        if batch is None:
            return None
        return batch[0], batch[1], (batch[2] if self.config.dataset in FLOW_DATASETS else None)

    def flow_step(self, batch, next_batch=None, fetch_losses=False, use_graph=True):
        """One PWC-Net update on `batch` = (img1, img2, flow, ...) or, unsupervised, (img1, img2, ...) (this rank's slice), overlapping
        the upload of `next_batch`; -> {global_step} + the FlowTrainGraph.losses() terms when fetch_losses.  All ranks must pass the
        same fetch_losses (the losses are all-reduced)."""
        g = self.graph
        self.global_step += 1
        lr = self._rate(self.global_step)
        if lr != self._lr:
            g.set_lr(lr)
            self._lr = lr
        g.feed(*self._flow_batch(batch))
        g.train_step(allreduce=self._allreduce(), use_graph=use_graph)
        if next_batch is not None:
            g.prefetch(*self._flow_batch(next_batch))
        res = {'global_step': self.global_step}
        if fetch_losses:
            res.update(g.losses(reduce=self._allreduce()))
        return res

    def save_flow(self, checkpoint_dir, epoch):
        """`pwcnet-<epoch>`: a TF V2 bundle of the pwcnet/* variables only (no global_step, no Adam slots) plus the same tensors as a
        native `.pt`, and the `checkpoint` state file.  epoch='best' writes pwcnet-best (the lowest validation EPE so far)."""
        if self.rank != 0:
            return
        base = 'pwcnet-%s' % epoch
        print(" [*] Saving PWC-Net to {}/{}".format(checkpoint_dir, base))
        self._write_checkpoint(checkpoint_dir, base, {k: v.cpu() for k, v in self.graph.export_params().items()}, None)

    def train_flow(self, config):
        """num_samples_train / batch_size steps per epoch for max_epochs epochs.  Every summary_freq steps rank 0 prints and writes
        the FlowTrainGraph.losses() terms (flow_loss and its parts); every save_freq epochs and after the last one it saves pwcnet-<epoch>.
        With config.validate every epoch ends with a validation: on Flying Chairs validate_flow(), rank 0 prints and writes
        `Validation EPE (flow)`; on a mask dataset validate_unsup(), `Validation unsupervised flow loss`.  pwcnet-best is saved whenever
        the value improves."""
        self.config = config
        self.build_flow_graph()
        g = self.graph
        if self.rank == 0:
            print("Number of PWC-Net params: {}".format(g.store.real_count()))
            print("-------------------------------------")
            print("Training PWC-Net ({} loss) on {}x{}, options {}".format(g.loss, g.H, g.W, dict(g.options._asdict())))
            print("-------------------------------------")
        w = self.collect_summaries()
        steps_per_epoch = self.train_steps_per_epoch
        batch = self.reader.batch(self.local_batch)
        for step in count(start=1):
            start_time = time.time()
            nxt = self.reader.batch(self.local_batch)
            fetch = step % config.summary_freq == 0
            res = self.flow_step(batch, next_batch=nxt, fetch_losses=fetch)
            batch = nxt
            if fetch and self.rank == 0:
                epoch = math.ceil(step / steps_per_epoch)
                print("Epoch: [%2d] [%5d/%5d] time: %4.4f/it flow_loss %4.4f"
                      % (epoch, step - (epoch - 1) * steps_per_epoch, steps_per_epoch, time.time() - start_time, res['flow_loss']))
                if w is not None:
                    for k in SUMMARY_KEYS[g.loss]:
                        w.add_scalar(k, res[k])
                    w.flush_step(res['global_step'])
            if step % steps_per_epoch == 0:
                epoch = step // steps_per_epoch
                last = epoch == config.max_epochs
                if epoch % config.save_freq == 0 or last:
                    self.save_flow(config.checkpoint_dir, epoch)
                if getattr(config, 'validate', False):
                    self._flow_validation_epoch_end(epoch)
                if last:
                    if self.rank == 0:
                        print("-------------------------------")
                        print("Training completed successfully")
                        print("-------------------------------")
                    break

    def _flow_validation_epoch_end(self, epoch):
        if self.config.dataset in FLOW_DATASETS:
            tag, val = "Validation EPE (flow)", self.validate_flow()
        else:
            tag, val = "Validation unsupervised flow loss", self.validate_unsup()
        if self.rank == 0:
            print("Epoch [{}] {}: {:.4f}".format(epoch, tag, val))
            if self.summary_writer is not None:
                self.summary_writer.add_scalar(tag, val)
                self.summary_writer.flush_step(epoch)
        if val < self.min_val_epe:                  # the same all-reduced value on every rank
            self.min_val_epe = val
            self.save_flow(self.config.checkpoint_dir, 'best')

    def validate_unsup(self):
        """The unsupervised objective on the val partition of a mask dataset -> the mean over its frame pairs of the pair's two
        directions' P + lambda_s * Sm (FlowTrainGraph.direction_objective).  The training graph's forward runs the val pairs in order
        (test_inputs at --test_temporal_shift and --test_crop), sharded over ranks like the evaluation; the sums are added on the device
        (pairs that only pad the last global batch are left out) and merged by one all-reduce."""
        g, cfg = self.graph, self.config
        n, GB, lb = self.num_samples_val, cfg.batch_size, self.local_batch
        tot = torch.zeros(2, dtype=torch.float64, device=self.device)
        it = self.dataset_reader.test_inputs(batch_size=GB, t_len=cfg.test_temporal_shift, test_crop=cfg.test_crop,
                                             partition='val').shard(self.rank, self.world, GB)
        try:
            for k in range(-(-n // GB)):
                batch = it.batch(lb)
                first = k * GB + self.rank * lb
                g.feed(batch[0], batch[1])
                g.forward()
                valid = min(lb, n - first)
                if valid > 0:
                    o = g.direction_objective()
                    tot[0] += o[:valid].sum() + o[lb:lb + valid].sum()
                    tot[1] += valid
        finally:
            it.close()
        d = _dist()
        if d is not None and self.world > 1:
            d.all_reduce(tot)
        s = tot.tolist()
        return s[0] / s[1] if s[1] else math.nan

    def validate_flow(self):
        """End-point error of the final flow on the val split -> mean over its pixels, in pixels of the 384x640 grid.  The training
        graph's forward runs the val pairs in order, sharded over ranks like the evaluation; the per-sample sums of FlowTrainGraph.epe
        are added over the batches on the device (pairs that only pad the last global batch are left out) and merged by one
        all-reduce."""
        g = self.graph
        n, GB, lb = self.num_samples_val, self.config.batch_size, self.local_batch
        tot = torch.zeros(4, dtype=torch.float64, device=self.device)
        it = self.dataset_reader.test_inputs(batch_size=GB).shard(self.rank, self.world, GB)
        try:
            for k in range(-(-n // GB)):
                batch = it.batch(lb)
                first = k * GB + self.rank * lb
                g.feed(batch[0], batch[1], batch[2])
                g.forward()
                valid = min(lb, n - first)
                if valid > 0:
                    tot += g.epe()[:valid].sum(0)
        finally:
            it.close()
        d = _dist()
        if d is not None and self.world > 1:
            d.all_reduce(tot)
        s = tot.tolist()
        return s[0] / s[2] if s[2] else math.nan
