"""FlowLearner: trains or fine-tunes PWC-Net (scope pwcnet) on Flying Chairs with the multi-scale flow loss (flow_train_graph.py), and
writes pwcnet-<epoch> checkpoints that --flow_ckpt of train.py, test_generator*.py, pretrain_recover.py and export_flow.py read.

It is AdversarialLearner's counterpart for the flow network: the same process setup (one process per GPU under torchrun, the global
batch sharded over ranks, one NCCL all-reduce of the flat gradient per step), reader, summaries and checkpoint writer.  The PWC-Net option
set is model_pwcnet._DEFAULT_PWCNET_TEST_OPTIONS, as for every other graph.
"""
import math
import time
from itertools import count

import torch

from .adversarial_learner import AdversarialLearner, FLOW_DATASETS, _dist
from .PWCNet import model_pwcnet
from .. import params_init
from ..flow_train_graph import FlowTrainGraph
from ..step_graph import PWC_H, PWC_W


def learning_rate_at(step, base, boundaries):
    """Rate of update number `step` (1-based): `base`, halved once for every boundary b < step (updates after the first b run at half
    the rate)."""
    return base * 0.5 ** sum(1 for b in boundaries if step > b)


class FlowLearner(AdversarialLearner):
    _lr = None                                          # the rate last written to the graph
    min_val_epe = math.inf

    def build_flow_graph(self):
        """FlowTrainGraph at img_height x img_width on the Flying Chairs 384x640 batches (the frames are resized on the device, the loss
        samples its targets from the 384x640 flow); parameters from --flow_ckpt when given, else params_init.init_pwcnet."""
        cfg = self.config
        if cfg.dataset not in FLOW_DATASETS:
            raise IOError('PWC-Net training needs a dataset with ground-truth flow (%s), got %s' % (', '.join(FLOW_DATASETS), cfg.dataset))
        self._init_dist()
        if cfg.batch_size % self.world:
            raise ValueError('batch_size must be divisible by the number of ranks')
        self.local_batch = cfg.batch_size // self.world
        self._pretrain = True                           # load_training_data: Flying Chairs' train pairs
        self.load_training_data()
        self.graph = FlowTrainGraph(cfg.img_height, cfg.img_width, self.local_batch, options=model_pwcnet._DEFAULT_PWCNET_TEST_OPTIONS,
                                    global_batch=cfg.batch_size, device=self.device, in_hw=(PWC_H, PWC_W),
                                    loss=getattr(cfg, 'flow_loss', 'multiscale'), weight_decay=getattr(cfg, 'weight_decay', 4e-4),
                                    lr=self._rate(1), beta1=cfg.beta1)
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

    def flow_step(self, batch, next_batch=None, fetch_losses=False, use_graph=True):
        """One PWC-Net update on `batch` = (img1, img2, flow, ...) (this rank's slice), overlapping the upload of `next_batch`;
        -> {global_step, flow_loss?, flow_loss_l6? .. flow_loss_l2?}.  All ranks must pass the same fetch_losses (the losses are
        all-reduced)."""
        g = self.graph
        self.global_step += 1
        lr = self._rate(self.global_step)
        if lr != self._lr:
            g.set_lr(lr)
            self._lr = lr
        g.feed(batch[0], batch[1], batch[2])
        g.train_step(allreduce=self._allreduce(), use_graph=use_graph)
        if next_batch is not None:
            g.prefetch(next_batch[0], next_batch[1], next_batch[2])
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
        flow_loss, flow_loss_l6 .. flow_loss_l2; every save_freq epochs and after the last one it saves pwcnet-<epoch>.  With
        config.validate every epoch ends with validate_flow(): rank 0 prints and writes `Validation EPE (flow)`, and pwcnet-best is saved
        whenever it improves."""
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
                    for k in ['flow_loss'] + ['flow_loss_l%d' % l for l in (6, 5, 4, 3, 2)]:
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
        epe = self.validate_flow()
        if self.rank == 0:
            print("Epoch [{}] Validation EPE (flow): {:.4f}".format(epoch, epe))
            if self.summary_writer is not None:
                self.summary_writer.add_scalar("Validation EPE (flow)", epe)
                self.summary_writer.flush_step(epoch)
        if epe < self.min_val_epe:                  # the same all-reduced value on every rank
            self.min_val_epe = epe
            self.save_flow(self.config.checkpoint_dir, 'best')

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
