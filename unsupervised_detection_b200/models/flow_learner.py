"""FlowLearner: trains or fine-tunes PWC-Net (scope pwcnet) on Flying Chairs with the multi-scale flow loss, or on the frame pairs of
DAVIS2016 / FBMS / SEGTRACK (or Flying Chairs) with the unsupervised loss (flow_train_graph.py), and writes pwcnet-<epoch> checkpoints
that --flow_ckpt of train.py, test_generator*.py, pretrain_recover.py and export_flow.py read.

It is AdversarialLearner's counterpart for the flow network: the same process setup (one process per GPU under torchrun, the global
batch sharded over ranks, one NCCL all-reduce of the flat gradient per step), reader, training loop, sharded validation pass, summaries
and checkpoint writer.  The PWC-Net option
set is model_pwcnet._DEFAULT_PWCNET_TEST_OPTIONS, as for every other graph.
"""
import math

from .adversarial_learner import AdversarialLearner, FLOW_DATASETS, MASK_DATASETS
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

    def build_flow_graph(self):
        """FlowTrainGraph at img_height x img_width on the 384x640 batches (the frames are resized on the device; the supervised losses
        sample their targets from the 384x640 flow); parameters from --flow_ckpt when given, else params_init.init_pwcnet.  The
        unsupervised loss also reads the training pairs of a mask dataset (--train_partition, --train_crop, the temporal shifts).  With
        --flow_aug every training batch is augmented on the device; sample b of rank r is global sample r * local_batch + b, so a
        data-parallel job draws the augmentation of one GPU running the global batch."""
        cfg = self.config
        loss = getattr(cfg, 'flow_loss', 'multiscale')
        ok = FLOW_DATASETS + (MASK_DATASETS if loss == 'unsupervised' else ())
        if cfg.dataset not in ok:
            raise IOError('PWC-Net training with the %s loss needs a dataset in %s, got %s' % (loss, ', '.join(ok), cfg.dataset))
        self._init_training_ranks()
        self._pretrain = True                           # load_training_data: Flying Chairs' train pairs
        self.load_training_data()
        self.graph = FlowTrainGraph(cfg.img_height, cfg.img_width, self.local_batch, options=model_pwcnet._DEFAULT_PWCNET_TEST_OPTIONS,
                                    global_batch=cfg.batch_size, device=self.device, in_hw=(PWC_H, PWC_W),
                                    loss=loss, weight_decay=getattr(cfg, 'weight_decay', 4e-4),
                                    lr=self._rate(1), beta1=cfg.beta1, smooth_weight=getattr(cfg, 'smooth_weight', 3.0),
                                    augment=getattr(cfg, 'flow_aug', False), sample_offset=self.rank * self.local_batch,
                                    ema_decay=self._ema_decay())
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

    def _resume(self):
        """AdversarialLearner._resume, then the learning rate of the next update."""
        out = super()._resume()
        self._lr = self._rate(self.global_step + 1)
        self.graph.set_lr(self._lr)
        return out

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
        native `.pt`, and the `checkpoint` state file.  epoch='best' writes pwcnet-best (the lowest validation EPE so far).  With
        --ema_decay each variable's moving average is there too, as <var>/ExponentialMovingAverage."""
        base = 'pwcnet-%s' % epoch
        self._write_checkpoint(checkpoint_dir, base, self.graph.export_params, None, "PWC-Net to {}/{}".format(checkpoint_dir, base))

    def train_flow(self, config):
        """PWC-Net training in _epoch_loop: the scalars are the FlowTrainGraph.losses() terms (flow_loss and its parts), the checkpoints
        pwcnet-<epoch> (save_flow).  With config.validate every epoch ends with a validation kept at its lowest in pwcnet-best: on Flying
        Chairs validate_flow(), logged as `Validation EPE (flow)`; on a mask dataset validate_unsup(), `Validation unsupervised flow
        loss`."""
        self.config = config
        self._kind = 'flow'
        self.build_flow_graph()
        g = self.graph

        def validate():
            if config.dataset in FLOW_DATASETS:
                tag, val = "Validation EPE (flow)", self.validate_flow()
            else:
                tag, val = "Validation unsupervised flow loss", self.validate_unsup()
            return val, "{}: {:.4f}".format(tag, val), tag
        self._epoch_loop(
            header=("Number of PWC-Net params: {}".format(g.store.real_count()),
                    "Training PWC-Net ({} loss) on {}x{}, options {}".format(g.loss, g.H, g.W, dict(g.options._asdict()))),
            step=lambda batch, nxt, fetch: self.flow_step(batch, next_batch=nxt, fetch_losses=fetch),
            progress=lambda r: ("flow_loss %4.4f" % r['flow_loss'], {k: r[k] for k in SUMMARY_KEYS[g.loss]}),
            epoch_end=lambda epoch: self._save_and_validate(epoch, self.save_flow, validate),
            banner="Training completed successfully")

    def validate_unsup(self):
        """The unsupervised objective on the val partition of a mask dataset -> the mean over its frame pairs of the pair's two
        directions' P + lambda_s * Sm (FlowTrainGraph.direction_objective).  The training graph's forward runs the val pairs of
        test_inputs at --test_temporal_shift and --test_crop in _val_sums."""
        g, cfg, lb = self.graph, self.config, self.local_batch

        def run(batch, first):
            g.feed(batch[0], batch[1])
            g.forward()

        def sums(valid):
            o = g.direction_objective()
            return o[:valid].sum() + o[lb:lb + valid].sum()
        it = self.dataset_reader.test_inputs(batch_size=cfg.batch_size, t_len=cfg.test_temporal_shift, test_crop=cfg.test_crop,
                                             partition='val')
        s = self._val_sums(it, 1, run, sums)
        n = self.num_samples_val                        # _val_sums scores each val pair on exactly one rank
        return s[0] / n if n else math.nan

    def validate_flow(self):
        """End-point error of the final flow on the val split -> mean over its pixels, in pixels of the 384x640 grid: the per-sample sums
        of FlowTrainGraph.epe after the training graph's forward, in _val_sums."""
        g = self.graph

        def run(batch, first):
            g.feed(batch[0], batch[1], batch[2])
            g.forward()
        s = self._val_sums(self.dataset_reader.test_inputs(batch_size=self.config.batch_size), 4, run, lambda valid: g.epe()[:valid].sum(0))
        return s[0] / s[2] if s[2] else math.nan
