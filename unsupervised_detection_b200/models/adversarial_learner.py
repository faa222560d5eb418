"""AdversarialLearner: the reference's learner surface (models/adversarial_learner.py:18-623) on the CUDA step graph.

Kept API: AdversarialLearner().train(config) / .setup_inference(config, aug_test=False) / .inference(sess) with the same
result keys (:617-619), plus .step() = one iteration of the loop body (:380-409) and .pretrain_recover(config) = pretraining of the
recover net on box-shaped occlusions (the pre-training behind --recover_ckpt that the reference's README describes), on PWC-Net's flow or
a dataset's ground-truth flow, with .validate_recover() = its held-out inpainting error.  With config.flow_dir set (not in the
reference), every graph takes a supplied flow field in place of PWC-Net's (CISGraph(flow_source='input')): training, validation IoU,
inference and the multi-crop ensemble, with no PWC-Net built and no --flow_ckpt read.  `sess` arguments are accepted and
ignored (there is no tf.Session).  Data parallelism (not in the reference): one process per GPU, the frame-pair batch is
sharded over ranks and the active network's flat gradient buffer is summed with ONE NCCL all-reduce per step
(SURVEY.md section 8e); clip / noise test / Adam then run identically on every rank.
"""
import math
import os
import time
from itertools import count

import numpy as np
import torch

from ..step_graph import CISGraph, PWC_H, PWC_W, box_sides
from .PWCNet import model_pwcnet
from ..data.synthetic import SyntheticReader
from .. import params_init
from .. import checkpoint as ckpt_io
from .. import flow_flags                               # defines --flow_dir for every script that drives the learner
from .utils.general_utils import compute_all_IoU


# CIS_PIPELINE=0 disables the cross-step software pipeline of the frozen flow network (see CISGraph.train_step)
PIPELINE = os.environ.get('CIS_PIPELINE', '1') != '0'
# datasets whose batches carry ground-truth flow (img1, img2, flow, names): recover-net pretraining with pretrain_flow=gt
FLOW_DATASETS = ('FLYINGCHAIRS',)
# datasets with masks; with a flow_dir their batches carry the supplied flow as a fifth element (img1, img2, seg1, names, flow)
MASK_DATASETS = ('DAVIS2016', 'FBMS', 'SEGTRACK')


def has_flow(dataset, flow_dir):
    """True when the batches of `dataset` carry flow: ground-truth flow (FLOW_DATASETS), or a mask dataset read with a flow_dir."""
    return dataset in FLOW_DATASETS or (dataset in MASK_DATASETS and bool(flow_dir))


def _dist():
    import torch.distributed as dist
    return dist if (dist.is_available() and dist.is_initialized()) else None


class AdversarialLearner(object):
    # Every attribute the methods read, with its initial value.  All are immutable, so they are declared on the class: a learner
    # made without __init__ (object.__new__, as host-side stubs do) reads the same defaults; assignments make instance attributes.
    config = graph = reader = val_reader = None
    global_step = 0
    _step = 0
    aug_test = False
    _inference = False                                  # test graphs: the dataset reader yields test inputs
    world, rank, local_rank, device = 1, 0, 0, None
    local_batch = num_samples_val = train_steps_per_epoch = val_steps_per_epoch = None
    min_val_iou = summary_writer = test_crops = None
    _gt_crops = _gt_small = None                        # device buffers of the multi-crop inference (_device_crops)
    _pretrain = False                                   # recover-net pretraining: datasets with flow (FLYINGCHAIRS) are accepted
    val_graph = None                                    # forward-only boxes graph of validate_recover, built on first use
    min_val_epe = math.inf
    _summary_img2 = None                                # frame 2 of the last summary step's batch (an input-flow graph has no img2)

    # ------------------------------------------------------------------------------------------------ data
    def load_training_data(self):
        """adversarial_learner.py:22-70.  Dataset readers are host-side code outside the accelerated path (SURVEY 8f-2);
        'SYNTHETIC' yields seeded frame pairs of the readers' shape.  Unknown datasets raise IOError like the reference.  A flow_dir
        needs a mask dataset (ValueError) and an existing directory (IOError)."""
        flow_flags.validate(self.config)
        ds = self.config.dataset
        if ds == 'SYNTHETIC':
            self.reader = SyntheticReader(PWC_H, PWC_W, seed=8964 + self.rank)
            self.num_samples_val = self.reader.val_samples
            return
        if ds == 'FLYINGCHAIRS' and self._pretrain:
            # frame pairs with ground-truth flow and no masks: recover-net pretraining only (train.py validates IoU on masks).  Training
            # reads the split's train pairs whatever --train_partition says, so that the val pairs stay held out.
            from ..data.flyingchairs_data_utils import FlyingChairsReader
            cfg = self.config
            self.dataset_reader = FlyingChairsReader(cfg.root_dir, num_threads=cfg.num_threads, seed=8964 + self.rank)
            self.reader = self.dataset_reader.image_inputs(batch_size=cfg.batch_size, train_crop=cfg.train_crop)
            self.num_samples_val = self.dataset_reader.val_samples
            return
        if ds in MASK_DATASETS:
            cfg = self.config
            if ds == 'DAVIS2016':
                from ..data.davis2016_data_utils import Davis2016Reader as Reader
            elif ds == 'FBMS':
                from ..data.fbms_data_utils import FBMS59Reader as Reader
                if self._inference and self.aug_test:
                    assert 'FBMS' in cfg.root_dir                              # adversarial_learner.py:542
            else:
                from ..data.segtrackv2_data_utils import SegTrackV2Reader as Reader
            rd = Reader(cfg.root_dir, max_temporal_len=cfg.max_temporal_len, min_temporal_len=cfg.min_temporal_len,
                        num_threads=cfg.num_threads, seed=8964 + self.rank, flow_dir=self.flow_dir())
            self.dataset_reader = rd
            if self._inference:
                self.reader = rd.test_inputs(batch_size=cfg.batch_size, t_len=cfg.test_temporal_shift, with_fname=True,
                                             test_crop=(1.0 if self.aug_test else cfg.test_crop), partition=cfg.test_partition)
                self.reader.val_samples = rd.val_samples
                if self.world > 1:      # batch-sharded evaluation (eval_dp.py): rank r reads its slice of every global batch
                    per_rank = 1 if self.aug_test else cfg.batch_size
                    self.reader.shard(self.rank, self.world, per_rank * self.world)
            else:
                self.val_reader = rd.test_inputs(batch_size=cfg.batch_size, t_len=cfg.test_temporal_shift, test_crop=cfg.test_crop,
                                                 partition='val').shard(self.rank, self.world, cfg.batch_size)
                self.num_samples_val = rd.val_samples
                self.reader = rd.image_inputs(batch_size=cfg.batch_size, train_crop=cfg.train_crop, partition=cfg.train_partition)
                self.reader.val_samples = self.num_samples_val
            if ds == 'FBMS':
                self.num_categories = rd.num_categories                       # :52
            return
        raise IOError("Dataset should be DAVIS2016 / FBMS / SEGTRACK")

    # ------------------------------------------------------------------------------------------------ graphs
    def flow_dir(self):
        """config.flow_dir: the directory of supplied .flo files, '' (or absent) = PWC-Net's flow."""
        return getattr(self.config, 'flow_dir', '') or ''

    def _flow_source(self):
        return 'input' if self.flow_dir() else 'pwc'

    def _init_dist(self):
        self.world, self.rank, self.local_rank = 1, 0, 0
        if int(os.environ.get('WORLD_SIZE', '1')) > 1:
            import torch.distributed as dist
            self.local_rank = int(os.environ.get('LOCAL_RANK', '0'))
            torch.cuda.set_device(self.local_rank)
            if not dist.is_initialized():
                dist.init_process_group('nccl', device_id=torch.device('cuda', self.local_rank))
            self.world, self.rank = dist.get_world_size(), dist.get_rank()
        self.device = 'cuda:%d' % self.local_rank
        torch.cuda.set_device(self.local_rank)

    def build_train_graph(self):
        """adversarial_learner.py:72-258: PWC-Net -> resize -> generator -> 3x recover -> losses -> two train ops."""
        cfg = self.config
        self._init_dist()
        if cfg.batch_size % self.world:
            raise ValueError('batch_size must be divisible by the number of ranks')
        self.local_batch = cfg.batch_size // self.world
        self.load_training_data()
        self.graph = CISGraph(cfg.img_height, cfg.img_width, self.local_batch, device=self.device, global_batch=cfg.batch_size,
                              flow_normalizer=cfg.flow_normalizer, cbn=cfg.cbn, epsilon=cfg.epsilon, beta1=cfg.beta1, with_pwc=True, train=True,
                              pwc_options=model_pwcnet._DEFAULT_PWCNET_TEST_OPTIONS, masks='generator', flow_source=self._flow_source())
        self.train_steps_per_epoch = int(math.ceil(cfg.num_samples_train / cfg.batch_size))
        self.val_steps_per_epoch = int(np.ceil(float(self.num_samples_val) / cfg.batch_size))
        self._init_params()

    # ------------------------------------------------------------------------------------------------ checkpoints
    @staticmethod
    def _is_ckpt(path):
        """True for a native `.pt` file or a TF V2 bundle prefix (`<prefix>.index` exists; `.index` / `.data-*` spellings ok)."""
        return bool(path) and (os.path.isfile(path) and path.endswith('.pt') or ckpt_io.is_bundle(ckpt_io.normalize_prefix(path)))

    @staticmethod
    def _read_ckpt(path, wanted, strict=True):
        """-> ({internal name: tensor}, global_step|None) from a native `.pt` file or a tf.train.Saver V2 bundle."""
        if os.path.isfile(path) and path.endswith('.pt'):
            st = torch.load(path, map_location='cpu')
            pr = st.get('params', st)
            if strict:
                miss = [k for k in wanted if k not in pr]
                if miss:
                    raise KeyError('checkpoint %s lacks %d variables, first %s' % (path, len(miss), miss[0]))
            return {k: pr[k] for k in wanted if k in pr}, st.get('global_step')
        prefix = ckpt_io.normalize_prefix(path)
        want = set(wanted)
        tfn = set(ckpt_io.to_tf_name(k, sep) for k in want for sep in ('//', '/')) | {'train_op/global_step', 'global_step'}
        # CIS_CKPT_NOVERIFY=1 skips the CRC-32C checks (block trailers, tensor payloads) -- an escape hatch for the first real
        # TF-written file, against which the reader's checksum handling has not been pinned yet
        verify = os.environ.get('CIS_CKPT_NOVERIFY') != '1'
        got, gs = ckpt_io.import_params(ckpt_io.read_bundle(prefix, names=lambda n: n in tfn, verify=verify), wanted, strict=strict)
        return {k: torch.from_numpy(np.array(v, dtype=np.float32)) for k, v in got.items()}, gs

    def _names(self, *scopes):
        g = self.graph
        stores = {'MaskNet': g.gen_store, 'FlownetS': g.rec_store, 'pwcnet': g.pwc_store}
        return [e[0] for sc in scopes for e in stores[sc].entries]

    def _init_params(self):
        cfg = self.config
        p = {}
        p.update(params_init.init_generator())
        p.update(params_init.init_recover())
        g = self.graph
        if g.flow_source != 'input':                                            # supplied flow: the graph has no PWC-Net
            p.update(self.flow_net_params())
        if getattr(cfg, 'resume_train', False):
            ck = cfg.full_model_ckpt if self._is_ckpt(cfg.full_model_ckpt) else self._latest_checkpoint(cfg.checkpoint_dir)
            assert ck, "Found no checkpoint to resume training!"               # :351
            # self.saver covers every trainable variable + global_step (:326-327); PWC-Net is frozen but trainable-typed
            # in the reference graph only through flow_saver, so it is optional here
            pr, gs = self._read_ckpt(ck, self._names('MaskNet', 'FlownetS'))
            p.update(pr)
            p.update(self._read_ckpt(ck, self._names('pwcnet'), strict=False)[0])
            self.global_step = int(gs or 0)
            print("Resumed training from model {}".format(ck))
        elif self._is_ckpt(getattr(cfg, 'recover_ckpt', '')):
            p.update(self._read_ckpt(cfg.recover_ckpt, self._names('FlownetS'))[0])  # recover_saver.restore, :354-358
            print("Recover net loaded from previous ckpt")
        else:
            print("No recover checkpoint found! Train Recover from Scratch")   # :360
        g.load_params(p)

    def flow_net_params(self):
        """PWC-Net's parameters for self.graph from config.flow_ckpt ('synthetic...' = the seeded stand-in) -> dict; IOError without
        a checkpoint."""
        fc = getattr(self.config, 'flow_ckpt', '')
        if fc.startswith('synthetic'):
            return params_init.init_pwcnet(self.graph.pwc_store.entries)
        if self._is_ckpt(fc):
            p = self._read_ckpt(fc, self._names('pwcnet'))[0]                    # flow_saver.restore, adversarial_learner.py:339-341
            print("Flow net loaded from {}".format(fc))
            return p
        raise IOError("Could not find flow ckpt file. Aborting.")              # adversarial_learner.py:343

    @staticmethod
    def _latest_checkpoint(d):
        """tf.train.latest_checkpoint(checkpoint_dir) (:349); falls back to the newest native `.pt` file."""
        if not d or not os.path.isdir(d):
            return None
        tfp = ckpt_io.latest_checkpoint(d)
        if tfp:
            return tfp
        c = [f for f in os.listdir(d) if f.startswith('model') and f.endswith('.pt')]
        return os.path.join(d, max(c, key=lambda f: os.path.getmtime(os.path.join(d, f)))) if c else None

    def save(self, sess, checkpoint_dir, step):
        """adversarial_learner.py:300-310: `saver.save(sess, checkpoint_dir/model[.best], global_step=step)` -- written as a
        tf.train.Saver V2 bundle (`model-<step>.index` + `.data-00000-of-00001` + the `checkpoint` state file, trainables +
        global_step, no Adam slots, max_to_keep=40 :327) that the reference itself can restore, plus the same tensors as a
        native torch file."""
        if self.rank != 0:
            return
        base = 'model.best' if step == 'best' else 'model-%s' % step
        print(" [*] Saving checkpoint to {}/model-{}".format(checkpoint_dir, step))
        params = {k: v.cpu() for k, v in self.graph.export_params().items()}
        self._write_checkpoint(checkpoint_dir, base, params, self.global_step)

    def save_recover(self, checkpoint_dir, epoch):
        """The recover net alone, as the reference's recover_saver covers it (adversarial_learner.py:329): `recover-<epoch>` as a TF V2
        bundle of the FlownetS variables (no global_step, no Adam slots) plus the same tensors as a native `.pt`, and the `checkpoint`
        state file.  train.py --recover_ckpt=<dir>/recover-<epoch> and a TF recover_saver.restore both read it.  epoch='best' writes
        recover-best (the lowest validation EPE so far), which later saves never delete."""
        if self.rank != 0:
            return
        base = 'recover-%s' % epoch
        print(" [*] Saving recover net to {}/{}".format(checkpoint_dir, base))
        params = {k: v.cpu() for k, v in self.graph.rec_store.export().items()}
        self._write_checkpoint(checkpoint_dir, base, params, None)

    def _write_checkpoint(self, checkpoint_dir, base, params, bundle_step):
        """<base>.pt + the <base> bundle (global_step in the bundle when bundle_step is not None); old entries beyond max_to_keep=40 go."""
        os.makedirs(checkpoint_dir, exist_ok=True)
        torch.save({'params': params, 'global_step': self.global_step}, os.path.join(checkpoint_dir, base + '.pt'))
        ckpt_io.write_bundle(os.path.join(checkpoint_dir, base), ckpt_io.export_params(params, bundle_step))
        for old in ckpt_io.update_checkpoint_state(checkpoint_dir, base, keep=40):
            for suf in ('.index', '.data-00000-of-00001', '.pt'):
                fp = os.path.join(checkpoint_dir, old + suf)
                if os.path.isfile(fp) and old not in ('model.best', 'recover-best', 'pwcnet-best'):
                    os.remove(fp)

    # ------------------------------------------------------------------------------------------------ stepping
    def _allreduce(self):
        d = _dist()
        if d is None or self.world == 1:
            return None
        return lambda t: d.all_reduce(t)     # sum: every rank's loss is already divided by the global batch

    def feed(self, img1, img2):
        """Host -> device copy of one batch of frame pairs [B,384,640,3] fp32 (CISGraph.feed)."""
        self.graph.feed(img1, img2)

    def prefetch(self, batch):
        """Start the host -> device copy of the NEXT batch on the copy stream so it overlaps the current step's kernels."""
        self.graph.prefetch(batch[0], batch[1])

    def step(self, batch=None, fetch_losses=None, use_graph=True, next_batch=None, summarize=False):
        """One iteration of the training loop body (adversarial_learner.py:380-409): picks train_recover_op or
        train_generator_op from the running step counter, consumes one batch, returns {global_step, loss_*?}."""
        cfg = self.config
        self._step += 1
        step = self._step
        sum_iters = cfg.iters_rec + cfg.iters_gen
        if step % sum_iters == 0:
            self.global_step += 1                                              # :382-384
        mode = 'R' if (step % sum_iters) < cfg.iters_rec else 'G'              # :386-389
        if batch is None:
            batch = self.reader.batch(self.local_batch)
        summarize = summarize and step % cfg.summary_freq == 0                 # :391-394 (same decision on every rank)
        if summarize:
            self._summary_img2 = batch[1]
        other_grads = self._train_on(mode, self._uploads(batch), self._uploads(next_batch), use_graph, summarize)
        res = {"global_step": self.global_step, "train_op": mode}
        fetch = fetch_losses if fetch_losses is not None else (step % cfg.summary_freq == 0)
        if fetch or summarize:
            # device -> host read; under data parallelism every rank holds its share of the global-batch losses (each is already
            # divided by the GLOBAL batch), so one SUM all-reduce of the four scalars gives every rank the true values -- all ranks
            # take this branch on the same steps
            L = self.graph.losses(full=summarize, reduce=self._allreduce())
            res["loss_recover"], res["loss_generator"] = L['recover'], L['generator']
        if summarize:
            self._write_step_summary(self.global_step, mode, other_grads, L)   # add_summary(results["summary"], gs), :403
        return res

    def _train_on(self, mode, batch, next_batch, use_graph, summarize):
        """Runs train op `mode` on `batch` (host tensors), overlapping the upload of `next_batch`; -> the other net's gradients
        when `summarize` (the summary pre-pass), else None."""
        g = self.graph
        if use_graph and next_batch is not None and not summarize and PIPELINE:
            # Software pipeline over steps: PWC-Net (frozen, parameter-independent) runs for `next_batch` on a second stream while
            # this step trains on `batch`, whose flow the previous call already left in the stage buffers.
            if g.stage_for is not batch[0]:
                self.feed(batch[0], batch[1])
                g.prime_pipeline()
            ready = g.feed_next(next_batch[0], next_batch[1])
            g.train_step(mode, allreduce=self._allreduce(), use_graph=True, pipeline=True, inputs_ready=ready)
            return None
        self.feed(batch[0], batch[1])
        other_grads = self._summary_prepass(mode) if summarize else None
        g.train_step(mode, allreduce=self._allreduce(), use_graph=use_graph)
        if next_batch is not None:
            self.prefetch(next_batch)          # overlaps this step's kernels; consumed by the next step() call
        return other_grads

    # ------------------------------------------------------------------------------------------------ summaries
    def collect_summaries(self):
        """adversarial_learner.py:260-298: opens the event file under checkpoint_dir (the Supervisor's logdir, :362-364) on
        rank 0.  Step summaries = 8 loss scalars, 6 images (first batch element), clipped-gradient histograms of every
        recover and generator variable; validation summary = "IoU on Validation"."""
        from ..summary import SummaryWriter
        cfg = self.config
        self.summary_writer = SummaryWriter(cfg.checkpoint_dir) if (self.rank == 0 and getattr(cfg, 'checkpoint_dir', '')) else None
        return self.summary_writer

    def _net_gradients(self, mode):
        """Host copy of one net's per-variable gradients as train_op returns them (loss_utils.py:28-32: clipped to +-0.2)."""
        store = self.graph.rec_store if mode == 'R' else self.graph.gen_store     # also works for a graph stub with the two stores
        flat = store.grad.detach().clamp(-0.2, 0.2).cpu().numpy()
        return [(name, flat[off:off + n]) for name, _, n, off, _ in store.entries]

    def _summary_prepass(self, mode):
        """The merged `step_sum` needs BOTH nets' gradients on a summary step (:283-289) although only one train op runs:
        evaluate the other net's gradient on the same batch and parameters before the optimiser step."""
        other = 'G' if mode == 'R' else 'R'
        g = self.graph
        g.forward()
        g.bwd[other].run()
        ar = self._allreduce()
        if ar is not None:
            ar(g.store(other).grad)
        torch.cuda.synchronize()
        return self._net_gradients(other)

    def _write_step_summary(self, gs, mode, other_grads, losses=None):
        """`losses`: the (already all-reduced) dict of CISGraph.losses(full=True); its four first-sample diagnostics
        (reconstruction_loss, ..., adversarial_learner.py:201-204) are those of rank 0's first sample."""
        w = self.summary_writer
        if w is None:
            return
        from .utils.flow_utils import flow_to_image_pm
        from .utils.general_utils import disambiguate_forw_back
        g = self.graph
        B = g.B
        for k, v in (losses if losses is not None else g.losses(full=True)).items():   # :262-263
            w.add_scalar(k, v)
        flow = g.flow.cpu().numpy()
        mask = g.mask.cpu().numpy()
        pred = g.pred.cpu().numpy()
        rec = pred[:B] * mask + flow * (1.0 - mask)                            # self.pred_flow, :251
        rec_c = pred[:B] * (1.0 - mask) + flow * mask                          # self.pred_flow_compl, :252 (the PRIMARY prediction, as the reference)
        w.add_image("input_image", g.image[:1].cpu().numpy())                  # :265-268
        w.add_image("next_image", (g.img2 if g.img2 is not None else self._summary_img2)[:1].cpu().numpy())
        flow_img = flow_to_image_pm(flow)
        w.add_image("masked_flow", flow_img * (1.0 - disambiguate_forw_back(mask)))   # :269-272
        w.add_image("PWC_Flow", flow_img)
        w.add_image("Rec_flow", flow_to_image_pm(rec))
        w.add_image("Rec_flow_compl", flow_to_image_pm(rec_c))
        grads = {mode: self._net_gradients(mode), ('G' if mode == 'R' else 'R'): other_grads}
        for m in ('R', 'G'):                                                   # :283-289, recover first
            for name, gv in grads[m]:
                w.add_histogram(ckpt_io.to_tf_name(name) + "/gradients", gv)
        w.flush_step(gs)

    def train(self, config):
        """adversarial_learner.py:312-420."""
        self.config = config
        self.build_train_graph()
        self.min_val_iou = -1.0e12
        if self.rank == 0:
            print("Number of params: {}".format(self.graph.param_count()))
            print("-------------------------------------")
            print("Training {} Recover and {} Generator".format(config.iters_rec, config.iters_gen))
            print("-------------------------------------")
        self.collect_summaries()
        batch = self.reader.batch(self.local_batch)
        for step in count(start=1):
            start_time = time.time()
            # the next batch (already decoded by the reader's background prefetch) is copied to the device on the side stream while this
            # step computes -- the same step(batch, next_batch=...) pattern bench.py's end-to-end arm measures
            nxt = self.reader.batch(self.local_batch)
            results = self.step(batch, summarize=True, next_batch=nxt)
            batch = nxt
            if step % config.summary_freq == 0 and self.rank == 0:
                train_epoch = math.ceil(step / self.train_steps_per_epoch)
                train_step = step - (train_epoch - 1) * self.train_steps_per_epoch
                print("Epoch: [%2d] [%5d/%5d] time: %4.4f/it loss_generator: %4.4f loss_recover %4.4f"
                      % (train_epoch, train_step, self.train_steps_per_epoch, time.time() - start_time,
                         results["loss_generator"], results["loss_recover"]))
            if step % self.train_steps_per_epoch == 0:
                train_epoch = int(step / self.train_steps_per_epoch)
                self.epoch_end_callback(None, None, train_epoch)
                if train_epoch == self.config.max_epochs:
                    if self.rank == 0:
                        print("-------------------------------")
                        print("Training completed successfully")
                        print("-------------------------------")
                    break

    def epoch_end_callback(self, sess, sv, epoch_num):
        """adversarial_learner.py:422-448: validation IoU, save best / every save_freq epochs."""
        validation_iou = 0.0
        vr = self.val_reader or self.reader
        for _ in range(self.val_steps_per_epoch):
            batch = vr.batch(self.local_batch)
            gt = batch[2]
            self.feed(*self._uploads(batch))
            self.graph.forward()
            masks = self.graph.mask.cpu().numpy()
            gtr = torch.nn.functional.interpolate(gt.permute(0, 3, 1, 2), size=masks.shape[1:3], mode='nearest').permute(0, 2, 3, 1).numpy()
            validation_iou += float(np.sum(compute_all_IoU(masks, gtr)))
        d = _dist()
        if d is not None and self.world > 1:
            t = torch.tensor([validation_iou], device=self.device)
            d.all_reduce(t)
            validation_iou = float(t)
        validation_iou /= self.val_steps_per_epoch * self.config.batch_size
        if self.rank == 0:
            w = self.summary_writer
            if w is not None:
                w.add_scalar("IoU on Validation", validation_iou)             # :296-298, :436-439
                w.flush_step(epoch_num)
            print("Epoch [{}] Validation IoU: {}".format(epoch_num, validation_iou))
        if validation_iou > self.min_val_iou:
            self.save(sess, self.config.checkpoint_dir, 'best')
            self.min_val_iou = validation_iou
        if epoch_num % self.config.save_freq == 0:
            self.save(sess, self.config.checkpoint_dir, epoch_num)

    # ------------------------------------------------------------------------------------------------ recover-net pretraining
    def build_pretrain_graph(self):
        """The recover step of adversarial_learner.py:72-258 with one random box per sample as the mask: PWC-Net -> resize -> box masks ->
        3x recover -> losses -> train_recover_op.  No generator runs.  config.box_min / box_max = box side range as fractions of the
        image sides (defaults 0.1 / 0.5).  config.pretrain_flow = 'pwc' (default: PWC-Net's flow of the frame pair) or 'gt' (the
        dataset's ground-truth flow, FLYINGCHAIRS, or the supplied flow of a mask dataset with config.flow_dir: no PWC-Net is built and
        --flow_ckpt is not read)."""
        cfg = self.config
        self._init_dist()
        if cfg.batch_size % self.world:
            raise ValueError('batch_size must be divisible by the number of ranks')
        self.local_batch = cfg.batch_size // self.world
        box = box_sides(getattr(cfg, 'box_min', 0.1), getattr(cfg, 'box_max', 0.5), cfg.img_height, cfg.img_width)
        gt = getattr(cfg, 'pretrain_flow', 'pwc') == 'gt'
        if gt and not has_flow(cfg.dataset, self.flow_dir()):
            raise ValueError('pretrain_flow=gt needs a dataset with ground-truth flow (%s) or a mask dataset (%s) with a flow_dir, got %s'
                             % (', '.join(FLOW_DATASETS), ', '.join(MASK_DATASETS), cfg.dataset))
        if self.flow_dir() and not gt:
            raise ValueError('a flow_dir replaces PWC-Net: recover-net pretraining on it needs pretrain_flow=gt')
        self._pretrain = True
        self.load_training_data()
        # sample_offset: sample b of rank r is global sample r * local_batch + b, so a DP job draws the boxes of one GPU running the global batch
        self.graph = CISGraph(cfg.img_height, cfg.img_width, self.local_batch, device=self.device, global_batch=cfg.batch_size,
                              flow_normalizer=cfg.flow_normalizer, cbn=cfg.cbn, epsilon=cfg.epsilon, beta1=cfg.beta1, with_pwc=True, train=True,
                              pwc_options=model_pwcnet._DEFAULT_PWCNET_TEST_OPTIONS, masks='boxes', box=box,
                              sample_offset=self.rank * self.local_batch, flow_source='input' if gt else 'pwc')
        self.train_steps_per_epoch = int(math.ceil(cfg.num_samples_train / cfg.batch_size))
        self._init_params()

    def _uploads(self, batch):
        """The two tensors of a reader batch (img1, img2, ... ) that the graph uploads: (frame 1, frame 2), or (frame 1, its flow) for an
        input-flow graph (a Flying Chairs batch is (img1, img2, flow, names), a mask dataset's with a flow_dir (img1, img2, seg1, names,
        flow))."""
        if batch is None:
            return None
        if getattr(self.graph, 'flow_source', 'pwc') != 'input':         # host-side graph stubs model the default graph
            return batch[0], batch[1]
        return batch[0], batch[4 if len(batch) > 4 else 2]

    def pretrain_step(self, batch, next_batch=None, fetch_losses=False, use_graph=True):
        """One pretraining iteration: train_recover_op on `batch` under box masks (one NCCL all-reduce of the recover gradient under
        torchrun); -> {global_step, loss_recover?, reconstruction_loss?, reconstruction_compl_loss?}.  All ranks must pass the same
        fetch_losses (the losses are all-reduced)."""
        self.global_step += 1
        self._train_on('R', self._uploads(batch), self._uploads(next_batch), use_graph, False)
        res = {"global_step": self.global_step}
        if fetch_losses:
            L = self.graph.losses(full=True, reduce=self._allreduce())
            res.update(loss_recover=L['recover'], reconstruction_loss=L['reconstruction_loss'],
                       reconstruction_compl_loss=L['reconstruction_compl_loss'])
        return res

    def pretrain_recover(self, config):
        """Pretrains the recover net (scope FlownetS) to inpaint optical flow under box-shaped occlusions, the pre-training the reference's
        README describes for --recover_ckpt.  num_samples_train / batch_size steps per epoch for max_epochs epochs; every summary_freq
        steps rank 0 prints the loss and writes the scalars recover / reconstruction_loss / reconstruction_compl_loss; every save_freq
        epochs and after the last one it saves recover-<epoch> (save_recover).  --flow_ckpt is mandatory unless pretrain_flow=gt,
        --recover_ckpt gives the starting weights (else the reference's initialisation).  config.validate: at every epoch end,
        validate_recover() on the val split; rank 0 prints and logs the EPE inside the boxes, and recover-best is saved whenever it
        improves."""
        self.config = config
        self.build_pretrain_graph()
        if self.rank == 0:
            print("Number of recover params: {}".format(self.graph.rec_store.real_count()))
            print("-------------------------------------")
            print("Pretraining Recover on box masks, sides {} px (h lo, h hi, w lo, w hi)".format(self.graph.box))
            print("-------------------------------------")
        w = self.collect_summaries()
        steps_per_epoch = self.train_steps_per_epoch
        batch = self.reader.batch(self.local_batch)
        for step in count(start=1):
            start_time = time.time()
            nxt = self.reader.batch(self.local_batch)
            fetch = step % config.summary_freq == 0
            results = self.pretrain_step(batch, next_batch=nxt, fetch_losses=fetch)
            batch = nxt
            if fetch and self.rank == 0:
                epoch = math.ceil(step / steps_per_epoch)
                print("Epoch: [%2d] [%5d/%5d] time: %4.4f/it loss_recover %4.4f"
                      % (epoch, step - (epoch - 1) * steps_per_epoch, steps_per_epoch, time.time() - start_time, results["loss_recover"]))
                if w is not None:
                    w.add_scalar("recover", results["loss_recover"])
                    w.add_scalar("reconstruction_loss", results["reconstruction_loss"])
                    w.add_scalar("reconstruction_compl_loss", results["reconstruction_compl_loss"])
                    w.flush_step(results["global_step"])
            if step % steps_per_epoch == 0:
                epoch = step // steps_per_epoch
                last = epoch == config.max_epochs
                if epoch % config.save_freq == 0 or last:
                    self.save_recover(config.checkpoint_dir, epoch)
                if getattr(config, 'validate', False):
                    self._validation_epoch_end(epoch)
                if last:
                    if self.rank == 0:
                        print("-------------------------------")
                        print("Pretraining completed successfully")
                        print("-------------------------------")
                    break

    def _validation_epoch_end(self, epoch):
        epe, epe_out = self.validate_recover()
        if self.rank == 0:
            print("Epoch [{}] Validation EPE (boxes): {:.4f} (outside the boxes: {:.4f})".format(epoch, epe, epe_out))
            if self.summary_writer is not None:
                self.summary_writer.add_scalar("Validation EPE", epe)
                self.summary_writer.flush_step(epoch)
        if epe < self.min_val_epe:                  # the same all-reduced value on every rank
            self.min_val_epe = epe
            self.save_recover(self.config.checkpoint_dir, 'best')

    def validate_recover(self):
        """Held-out inpainting error of the recover net -> (EPE inside the boxes, EPE outside them), means over the pixels of the val
        split in pixels of the 384x640 grid.  A forward-only boxes graph with the training graph's weights runs the val pairs in order,
        sharded over ranks like the evaluation; its step counter stays 0 and each batch's sample_offset is its global val index, so
        every call scores the same boxes.  cis_masked_epe's per-sample sums are added over the batches on the device (pairs that only
        pad the last global batch are left out) and merged by one all-reduce."""
        cfg, g = self.config, self.graph
        if self.val_graph is None:
            self.val_graph = CISGraph(cfg.img_height, cfg.img_width, self.local_batch, device=self.device, global_batch=cfg.batch_size,
                                      flow_normalizer=cfg.flow_normalizer, cbn=cfg.cbn, epsilon=cfg.epsilon, with_pwc=True, train=False,
                                      pwc_options=model_pwcnet._DEFAULT_PWCNET_TEST_OPTIONS, masks='boxes', box=g.box,
                                      flow_source=g.flow_source)
        vg = self.val_graph
        vg.load_params(g.export_params())
        n, GB, lb = self.num_samples_val, cfg.batch_size, self.local_batch
        tot = torch.zeros(4, dtype=torch.float64, device=self.device)
        it = self.dataset_reader.test_inputs(batch_size=GB).shard(self.rank, self.world, GB)     # a fresh ordered pass every call
        try:
            for k in range(-(-n // GB)):
                batch = it.batch(lb)
                first = k * GB + self.rank * lb
                vg.set_sample_offset(first)
                vg.feed(*self._uploads(batch))
                vg.forward()
                valid = min(lb, n - first)
                if valid > 0:
                    tot += vg.masked_epe()[:valid].sum(0)
        finally:
            it.close()
        d = _dist()
        if d is not None and self.world > 1:
            d.all_reduce(tot)
        s = tot.tolist()
        return tuple(e / m * cfg.flow_normalizer if m else math.nan for e, m in ((s[0], s[2]), (s[1], s[3])))

    # ------------------------------------------------------------------------------------------------ inference
    def build_test_graph(self):
        """adversarial_learner.py:450-523: PWC-Net -> resize -> generator -> recover (forward only)."""
        cfg = self.config
        self._init_dist()
        self.local_batch = cfg.batch_size
        self._inference = True
        self.load_training_data()
        self.graph = CISGraph(cfg.img_height, cfg.img_width, self.local_batch, device=self.device, flow_normalizer=cfg.flow_normalizer,
                              cbn=cfg.cbn, epsilon=cfg.epsilon, with_pwc=True, train=False,
                              pwc_options=model_pwcnet._DEFAULT_PWCNET_TEST_OPTIONS, masks='generator', flow_source=self._flow_source())
        self.test_samples = self.reader.val_samples
        self.test_iterator = self.reader

    def build_aug_test_graph(self):
        """adversarial_learner.py:525-592: multi-crop ensemble, batch 1 per crop (the four crops are batched here)."""
        self.test_crops = [0.85, 0.9, 0.95, 1.0]
        print("Evaluating the following crops {}".format(self.test_crops))
        cfg = self.config
        self._init_dist()
        self.local_batch = len(self.test_crops)
        self._inference = True
        self.load_training_data()
        self.graph = CISGraph(cfg.img_height, cfg.img_width, self.local_batch, device=self.device, flow_normalizer=cfg.flow_normalizer,
                              with_pwc=True, train=False, pwc_options=model_pwcnet._DEFAULT_PWCNET_TEST_OPTIONS, masks='generator', flow_source=self._flow_source())
        self.test_samples = self.reader.val_samples
        self.test_iterator = self.reader

    def setup_inference(self, config, aug_test=False):
        """adversarial_learner.py:594-604."""
        self.config = config
        self.aug_test = aug_test
        if self.aug_test:
            self.build_aug_test_graph()
        else:
            self.build_test_graph()

    def restore(self, ckpt_file):
        """test_generator.py:45-58: restores ALL trainables (incl. PWC-Net) from one checkpoint (TF V2 bundle or native `.pt`).  An
        input-flow graph has no PWC-Net, so its variables are neither needed nor read."""
        if ckpt_file.startswith('synthetic'):
            p = {}
            p.update(params_init.init_generator())
            p.update(params_init.init_recover())
            p.update(params_init.init_pwcnet(self.graph.pwc_store.entries))
        elif self._is_ckpt(ckpt_file):
            p = params_init.init_recover()          # the mask path does not read the recover net; restored when present
            p.update(self._read_ckpt(ckpt_file, self._names('MaskNet', 'pwcnet'))[0])
            p.update(self._read_ckpt(ckpt_file, self._names('FlownetS'), strict=False)[0])
        else:
            raise IOError("Checkpoint file not found")                         # test_generator.py:58
        self.graph.load_params(p)

    def _device_crops(self, img1, img2, gt):
        """Multi-crop test-time augmentation on the device: host [1,Hs,Ws,C] tensors -> g.img1 / g.img2 rows (one per crop) and the
        nearest-resized ground-truth crops [ncrop,H,W,1] (numpy).  Same geometry and interpolation as data/crops.central_crops.  For an
        input-flow graph img2 is frame 1's flow [1,Hs,Ws,2]: its crops go to g.flow_full with the vectors scaled to the resize
        (cis_crop_resize_flow_f32: rows by Hs/ch, columns by Ws/cw)."""
        from ..data.davis2016_data_utils import central_crop_box
        from .. import _lib
        g = self.graph
        g.pipeline_drain()
        dev = g.img1.device
        st = torch.cuda.current_stream().cuda_stream
        hs, ws = int(img1.shape[1]), int(img1.shape[2])
        d1, d2, dg = img1.to(dev, non_blocking=True), img2.to(dev, non_blocking=True), gt.to(dev, non_blocking=True)
        nc = len(self.test_crops)
        if self._gt_crops is None or self._gt_crops.shape[0] != nc:
            self._gt_crops = torch.empty(nc, hs, ws, 1, dtype=torch.float32, device=dev)
            self._gt_small = torch.empty(nc, g.H, g.W, 1, dtype=torch.float32, device=dev)
        for i, c in enumerate(self.test_crops):
            y0, x0, ch, cw = central_crop_box(hs, ws, c)
            frames = [(d1, g.img1[i], 3)] + ([(d2, g.img2[i], 3)] if g.img2 is not None else [])
            for src, dst, C_ in frames + [(dg, self._gt_crops[i], 1)]:
                _lib.call('cis_crop_resize_bilinear_f32', src.data_ptr(), hs, ws, C_, y0, x0, ch, cw, dst.data_ptr(), hs, ws, st)
            if g.img2 is None:
                _lib.call('cis_crop_resize_flow_f32', d2.data_ptr(), hs, ws, y0, x0, ch, cw, g.flow_full[i].data_ptr(), hs, ws, hs / ch, ws / cw,
                          st)
        _lib.call('cis_resize_nn_f32', self._gt_crops.data_ptr(), nc, hs, ws, 1, self._gt_small.data_ptr(), g.H, g.W, st)
        self._keep_crop_src = (d1, d2, dg)
        return self._gt_small.cpu().numpy()

    def inference(self, sess=None, batch=None):
        """adversarial_learner.py:606-623 -> dict with the reference's keys (numpy arrays)."""
        g = self.graph
        if batch is None:
            batch = self.reader.batch(1 if self.aug_test else self.local_batch)
        (img1, img2), gt, names = self._uploads(batch), batch[2], batch[3]
        H, W = g.H, g.W
        if self.aug_test:
            # crops [0.85,0.9,0.95,1.0] of ONE frame pair, each resized back to 384x640 (davis2016_data_utils.py:328-354): the frame
            # pair is uploaded once and cut / resized on the device (cis_crop_resize_bilinear_f32) straight into the network inputs
            gtr = self._device_crops(img1[:1], img2[:1], gt[:1])
            g.forward_masks(use_graph=True)      # the multi-crop graph of the reference outputs masks only (:525-592)
        else:
            self.feed(img1, img2)
            g.forward()
            gtr = torch.nn.functional.interpolate(gt.permute(0, 3, 1, 2), size=(H, W), mode='nearest').permute(0, 2, 3, 1).numpy()
        masks = g.mask.cpu().numpy()
        if self.aug_test:
            outs = {'pred_masks': {}, 'gt_masks': {}, 'img_1s': {}}
            image = g.image.cpu().numpy()
            for i, c in enumerate(self.test_crops):
                outs['pred_masks'][c], outs['gt_masks'][c], outs['img_1s'][c] = masks[i], gtr[i], image[i]
            return {'outs': outs, 'img_fname': np.array(names[0].encode())}
        return {'gen_masks': masks, 'pred_flow': g.pred[:g.B].cpu().numpy(), 'input_image': g.image.cpu().numpy(),
                'gt_flow': g.flow.cpu().numpy(), 'gt_masks': gtr, 'img_fname': np.array([n.encode() for n in names])}
