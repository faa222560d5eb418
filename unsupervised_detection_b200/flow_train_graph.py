"""PWC-Net training step as static launch lists: tfoptflow's multi-scale objective on Flying Chairs-style (img1, img2, ground-truth flow)
batches, the full PWC-Net backward of PWCNetBuilder(trainable=True), and TF-Adam with L2 weight decay on the conv kernels.

The objective, as defined here (restated from the published tfoptflow / NVlabs PWC-Net training recipe; it is not checked against
TensorFlow): with flow_l the refined fp32 flow of level l = 6..2 and G the ground-truth flow at the network input size,
    L = sum_l alpha_l * (1/B) sum_b sum_pixels rho(flow_l - g_l)  +  (gamma/2) * sum_{kernels} ||w||^2,
    g_l = resize_bilinear_legacy(G, h_l, w_l) / 2^l,   rho = ||d||_2 ('multiscale') or (|d0| + |d1| + eps)^q ('robust').
B is the global batch, so that one SUM all-reduce of the flat gradient gives every rank the gradient of the global-batch loss.  The
L2 term is applied by the optimiser (cis_adam_l2) and is not part of losses().

loss='unsupervised' needs no ground truth (restated from UnFlow's published recipe; it is not checked against any other
implementation): the network runs on 2B pairs, the B pairs (img1, img2) and then the same pairs swapped, and with P_n the
occlusion-masked census term and Sm_n the edge-aware second-order smoothness of direction n's final flow (cis_unsup_flow_loss in
include/cis_b200.h states both),
    L = (1/GB) sum over the 2B directions of (P_n + lambda_s * Sm_n),   P_n = sum_p M psi / (H W),   Sm_n = sum_p sum_a w_a s_a / (H W).
GB is the global batch in pairs.  The occlusion mask M compares each direction's flow with its partner's and carries no gradient.

One step: pack the images (+0.5, adapt_x) -> PWC-Net forward -> loss forward (per-sample, per-level fp64 sums) -> seed (zero the level
gradients, loss backward into the five level-flow gradients) -> the builder's reverse tape -> fixed-order weight-gradient reduction ->
[one all-reduce] -> cis_adam_l2 -> re-pack of the bf16 operands.  The images carry no gradient dependency, so no conv1a data gradient is
emitted.  The unsupervised step seeds only the final flow: the loss backward writes d L / d flow at H x W, and the transpose of the
final x4 resize carries it into the level-2 flow gradient; levels 3-6 get theirs from the reverse tape alone.

augment=True (supervised losses only) puts a random affine and photometric augmentation in front of that step, restated from the
FlowNet / PWC-Net papers' description (cis_flow_aug_params and cis_flow_augment in include/cis_b200.h define it; the ranges, AUG_RANGES
below, are chosen here).  Its parameters are drawn on the device from a counter hash of (seed, the Adam step, the global sample index):
CUDA-graph replays draw new ones with no host involvement, and a data-parallel job with sample_offset = rank * batch draws what one GPU
running the global batch draws.  The step's resize, pack and loss then read the augmented copies of the uploaded batch; forward() copies
the batch unchanged into those buffers, so validation and epe() see the frames as uploaded.
"""
import ctypes as C

import torch

from . import _lib
from .engine import Act, Builder, ParamStore, Plan, averaged_weights, check_ema_decay
from .step_graph import UploadSlots, capture_plans

LEVELS = (6, 5, 4, 3, 2)                          # level i of the loss kernels is pyramid level LEVELS[i]
ALPHAS = (0.32, 0.08, 0.02, 0.01, 0.005)          # alpha_l for l = 6..2
WEIGHT_DECAY = 4e-4                               # gamma
ROBUST_EPS, ROBUST_Q = 0.01, 0.4
SMOOTH_WEIGHT = 3.0                               # lambda_s of the unsupervised loss: UnFlow's second-order weight, not tuned here
FLOW_LOSSES = ('multiscale', 'robust', 'unsupervised')
# augment=True: the default ranges of CisFlowAug (include/cis_b200.h states what each one draws)
AUG_RANGES = dict(scale=(0.9, 2.0), rotate=(-17.0, 17.0), translate=(-0.2, 0.2), rel_scale=(0.95, 1.05), rel_rotate=(-3.0, 3.0),
                  rel_translate=(-0.03, 0.03), color=(0.5, 2.0), contrast=(-0.8, 0.4), brightness=0.2, gamma=(0.7, 1.5), noise=(0.0, 0.04))
AUG_SEED = 8964


def flow_aug_ranges(**changes):
    """A CisFlowAug holding AUG_RANGES with `changes` (field name -> value) applied."""
    r = _lib.CisFlowAug()
    for k, v in dict(AUG_RANGES, **changes).items():
        if k not in AUG_RANGES:
            raise ValueError('unknown augmentation range %r' % k)
        if isinstance(v, tuple):
            getattr(r, k)[:] = [float(x) for x in v]
        else:
            setattr(r, k, float(v))
    return r


def check_size(H, W):
    """ValueError unless H and W are multiples of 64 (PWC-Net's six stride-2 levels) and at least 128 (the warp + cost volume needs
    level 6 to be at least 2x2)."""
    if H < 128 or W < 128 or H % 64 or W % 64:
        raise ValueError('PWC-Net training needs H, W multiples of 64 and at least 128, got %dx%d' % (H, W))


def kernel_segments(store):
    """[(start, end)] of the variables named */kernel in a ParamStore's flat buffer: where cis_adam_l2 applies the weight decay."""
    return [(off, off + n) for name, _, n, off, _ in store.entries if name.endswith('/kernel')]


class FlowTrainGraph(object):
    """One PWC-Net training step for a fixed (batch, H x W) geometry.

    options: PWC-Net options (the reference's keys; None = model_pwcnet._DEFAULT_PWCNET_TEST_OPTIONS).  global_batch: the batch of the
    whole data-parallel job (default: batch).  in_hw: size of the uploaded frames and flow (default H x W); when it differs, the frames
    are resized to H x W on the device and the loss samples its targets from the uploaded flow, its vectors scaled to the H x W grid.
    loss: 'multiscale', 'robust' or 'unsupervised'; alphas, weight_decay, eps, q: the objective's constants; smooth_weight: lambda_s of
    the unsupervised loss; lr, beta1, beta2, adam_eps: TF-Adam.  With loss='unsupervised' the network batch is 2 * batch (forward pairs,
    then backward pairs) and self.flow holds both halves; the ground truth is only read by epe().
    augment: train_step augments each uploaded batch at in_hw before the step (supervised losses only); aug_ranges: a CisFlowAug
    (flow_aug_ranges(); None = AUG_RANGES); sample_offset: the global index of this rank's first sample (rank * batch under data parallelism).
    ema_decay: 0 (the default) keeps no moving average; 0 < ema_decay < 1 gives the store a shadow that one cis_ema_update after
    cis_adam_l2 updates every step (averaged(), export_params())."""

    def __init__(self, H, W, batch, options=None, global_batch=None, device='cuda', in_hw=None, loss='multiscale', alphas=ALPHAS,
                 weight_decay=WEIGHT_DECAY, eps=ROBUST_EPS, q=ROBUST_Q, lr=1e-4, beta1=0.9, beta2=0.999, adam_eps=1e-8, name='pwcnet',
                 smooth_weight=SMOOTH_WEIGHT, augment=False, aug_ranges=None, sample_offset=0, ema_decay=0.0):
        from .models.PWCNet.model_pwcnet import PWCNetBuilder
        check_size(H, W)
        check_ema_decay(ema_decay)
        if loss not in FLOW_LOSSES:
            raise ValueError('loss must be one of %s, got %r' % (FLOW_LOSSES, loss))
        if len(alphas) != 5:
            raise ValueError('alphas: one weight per level 6..2, got %r' % (alphas,))
        if not smooth_weight >= 0:
            raise ValueError('smooth_weight must be >= 0, got %r' % (smooth_weight,))
        if augment and loss == 'unsupervised':
            raise ValueError('augment=True is for the supervised losses: the unsupervised loss scores the frames themselves')
        if sample_offset < 0:
            raise ValueError('sample_offset must be >= 0, got %r' % (sample_offset,))
        _lib.load()
        self.H, self.W, self.B = H, W, batch
        self.GB = global_batch or batch
        self.in_hw = ih, iw = tuple(in_hw or (H, W))
        self.dev = device
        self.loss, self.alphas, self.weight_decay = loss, tuple(float(a) for a in alphas), float(weight_decay)
        self.smooth_weight = float(smooth_weight)
        unsup = loss == 'unsupervised'
        B = batch
        N = 2 * B if unsup else B                           # the network batch
        self.store = ParamStore(device)
        self.pwc = PWCNetBuilder(self.store, name, trainable=True, options=options)
        self.options = self.pwc.options
        self.store.finalize(True)
        self.step_state = torch.zeros(1, dtype=torch.int64, device=device)      # TF-Adam's beta-power step
        self.lr = torch.full((1,), float(lr), dtype=torch.float32, device=device)   # read by cis_adam_l2 when it runs (set_lr)
        bld = Builder(device)
        self.bld = bld
        P = bld.fwd
        f32 = bld.f32
        self.img1, self.img2, self.gt = f32(B, ih, iw, 3), f32(B, ih, iw, 3), f32(B, ih, iw, 2)
        self.inputs = (self.img1, self.img2, self.gt)       # the three device buffers one batch upload writes
        self.augment, self.sample_offset = bool(augment), int(sample_offset)
        self.aug, self.copy_in = Plan('aug_P'), Plan('copy_P')
        if self.augment:
            # the step reads augmented copies of the upload: aug draws each sample's parameters and writes them; copy_in (forward())
            # writes the upload unchanged
            self.aug_ranges = aug_ranges if aug_ranges is not None else flow_aug_ranges()
            self.aug_seed = AUG_SEED
            self.aug_params = torch.zeros(B, _lib.FLOW_AUG_ROW, dtype=torch.float32, device=device)
            self.batch = (f32(B, ih, iw, 3), f32(B, ih, iw, 3), f32(B, ih, iw, 2))
            self.aug.keep += [self.aug_ranges, self.aug_params]
            self.aug.add('cis_flow_aug_params', C.byref(self.aug_ranges), B, ih, iw, self.sample_offset, self.step_state.data_ptr(),
                         self.aug_seed, self.aug_params.data_ptr())
            self.aug.add('cis_flow_augment', *(t.data_ptr() for t in self.inputs), self.aug_params.data_ptr(), B, ih, iw,
                         *(t.data_ptr() for t in self.batch))
            for dst, src in zip(self.batch, self.inputs):
                self.copy_in.add_py(lambda d=dst, s=src: d.copy_(s), 'copy')
        else:
            self.batch = self.inputs
        # the images carry no gradient dependency: the backward emits conv1a's weight gradient but no data gradient
        i1, i2 = Act(N, H, W, 3, device, name='img1_8'), Act(N, H, W, 3, device, name='img2_8')
        self.img_acts = bld.hold((i1, i2))
        src = self.batch[:2]
        if (ih, iw) != (H, W):
            src = (f32(B, H, W, 3), f32(B, H, W, 3))
            for a, b in zip(self.batch[:2], src):
                P.add('cis_resize_bilinear_f32', a.data_ptr(), B, ih, iw, 3, b.data_ptr(), H, W, 1.0)
        if unsup:
            # network pairs n < B: (img1, img2); n >= B: (img2, img1) -- each frame packed into one half of each image Act
            half = B * H * W * i1.pitch * i1.buf.element_size()
            for a, b in ((i1, src), (i2, src[::-1])):
                P.add('cis_pack_f32_to_bf16', b[0].data_ptr(), B * H * W, 3, 0.5, a.ptr, 8, 0)
                P.add('cis_pack_f32_to_bf16', b[1].data_ptr(), B * H * W, 3, 0.5, a.ptr + half, 8, 0)
        else:
            for a, b in zip(src, (i1, i2)):
                P.add('cis_pack_f32_to_bf16', a.data_ptr(), B * H * W, 3, 0.5, b.ptr, 8, 0)      # adapt_x: img + 0.5
        self.flow = f32(N, H, W, 2)                          # the network's output: the level-2 flow x4, at H x W
        self.pwc.build(bld, i1, i2, self.flow)
        if unsup:
            seed, seeds = self._plan_unsup_loss(P, src)
        else:
            seed, seeds = self._plan_multiscale_loss(P, eps, q)
        self.fwd = P
        layers = self.pwc.all_layers()
        self.bwd = bld.backward_plan('P', seed, seeds, layers)
        # ---- TF-Adam + L2 on the kernels (biases are not decayed)
        self.kernel_seg = kernel_segments(self.store)
        self._seg = torch.tensor([v for s in self.kernel_seg for v in s], dtype=torch.int64, device=device)
        st = self.store
        self.adam = Plan('adam_P')
        self.adam.keep.append(self._seg)
        self.adam.add('cis_adam_l2', st.flat.data_ptr(), st.m.data_ptr(), st.v.data_ptr(), st.grad.data_ptr(), st.size, self._seg.data_ptr(),
                      len(self.kernel_seg), self.weight_decay, self.lr.data_ptr(), float(beta1), float(beta2), float(adam_eps),
                      self.step_state.data_ptr())
        if ema_decay:
            st.add_shadow()
            self.adam.add('cis_ema_update', st.shadow.data_ptr(), st.flat.data_ptr(), st.size, ema_decay, self.step_state.data_ptr())
        # ---- bf16 operands (forward and data-gradient orientation), after backward planning decided what is needed
        pack = Plan('pack_P')
        for L in layers:
            L.plan_pack(pack, dgrad=True)
        self.pack = pack.batch_param_ops(device)
        self._dirty = True
        # held-out end-point error (epe): an all-ones mask, the prediction on the ground truth's grid, fixed-order sums
        self.epe_sums = torch.zeros(B, 4, dtype=torch.float64, device=device)
        self._epe_scratch = torch.zeros(B * 256, dtype=torch.float64, device=device)
        self._ones = torch.ones(B, ih, iw, dtype=torch.float32, device=device)
        self._pred_gt_grid = self.flow if (ih, iw) == (H, W) else torch.zeros(B, ih, iw, 2, dtype=torch.float32, device=device)
        # ---- device-only state, made on first use (a FlowTrainGraph is also built with device='cpu' to inspect its plans)
        self.graphs = {}
        self._copy = None                   # stream of the batch uploads (prefetch)
        self._uploads = UploadSlots(self.inputs, self._copy_stream)

    def _plan_multiscale_loss(self, P, eps, q):
        """Loss forward into P; -> (the seed Plan, the Acts it seeds)."""
        B, H, W, (ih, iw), device = self.B, self.H, self.W, self.in_hw, self.dev
        # ---- loss forward: per-sample, per-level sums of rho (fp64, fixed order)
        pyr = _lib.CisFlowPyr()
        for i, l in enumerate(LEVELS):
            g = self.pwc.flows_bf[l].get_grad()
            pyr.flow[i], pyr.grad[i], pyr.pitch[i], pyr.c_off[i] = self.pwc.flows[l].data_ptr(), g.ptr, g.pitch, g.c_off
            pyr.accumulate[i] = 0            # the loss backward writes first; up_flow's data gradient then accumulates (l >= 3)
            pyr.weight[i] = self.alphas[i] / self.GB
        self.pyr = pyr
        self.sums = torch.zeros(B, 5, dtype=torch.float64, device=device)
        self._scratch = torch.zeros(5 * B * 64, dtype=torch.float64, device=device)
        self._loss_args = (self.batch[2].data_ptr(), B, H, W, ih, iw, H / ih, W / iw, 1 if self.loss == 'robust' else 0, float(eps), float(q))
        P.keep.append(pyr)
        P.add('cis_flow_multiscale_loss', C.byref(pyr), *self._loss_args, self._scratch.data_ptr(), self.sums.data_ptr())
        # ---- backward: zero the DenseNet level gradients, seed the five level-flow gradients, reverse tape, weight-gradient reduction
        seed = Plan('seed_P')
        for g in self.pwc.level_grad.values():
            seed.zero(g)
        seed.keep.append(pyr)
        seed.add('cis_flow_multiscale_loss_bwd', C.byref(pyr), *self._loss_args)
        return seed, [self.pwc.flows_bf[l] for l in LEVELS]

    def _plan_unsup_loss(self, P, frames):
        """Unsupervised loss forward into P, on the fp32 frames at H x W; -> (the seed Plan, the Acts it seeds)."""
        from .models.PWCNet.model_pwcnet import FLOW_PRED_LVL
        B, H, W, f32 = self.B, self.H, self.W, self.bld.f32
        N = 2 * B
        # per-direction {sum M psi, sum w s} (fp64, fixed order); T~, M and M psi'(c) per pixel for the backward
        self.sums = torch.zeros(N, 2, dtype=torch.float64, device=self.dev)
        self._scratch = torch.zeros(2 * N * 64, dtype=torch.float64, device=self.dev)
        self.warped, self.mask, self.coef = f32(N, H, W), f32(N, H, W), f32(N, H, W)
        self._loss_args = (self.flow.data_ptr(), frames[0].data_ptr(), frames[1].data_ptr(), B, H, W)
        P.add('cis_unsup_flow_loss', *self._loss_args, self.warped.data_ptr(), self.mask.data_ptr(), self.coef.data_ptr(),
              self._scratch.data_ptr(), self.sums.data_ptr())
        # ---- backward: zero the DenseNet level gradients, d L / d flow at H x W, the transpose of the final x4 resize into the level-2
        # flow gradient.  Only that level is seeded: the levels 3-6 flow gradients are first written (not added to) by up_flow's data
        # gradient on the reverse tape.
        seed = Plan('seed_P')
        for g in self.pwc.level_grad.values():
            seed.zero(g)
        self.dflow = f32(N, H, W, 2)
        norm = float(self.GB * H * W)
        seed.add('cis_unsup_flow_loss_bwd', *self._loss_args, self.warped.data_ptr(), self.coef.data_ptr(), 1.0 / norm,
                 self.smooth_weight / norm, self.dflow.data_ptr())
        fb = self.pwc.flows_bf[FLOW_PRED_LVL]
        fg, s = fb.get_grad(), 2 ** FLOW_PRED_LVL
        seed.add('cis_resize_f32_bwd_to_bf16_scaled', self.dflow.data_ptr(), N, H, W, 2, H // s, W // s, fg.ptr, fg.pitch, float(s))
        return seed, [fb]

    # ------------------------------------------------------------------------------------------------ parameters
    def load_params(self, params):
        """params: dict name -> tensor with the pwcnet/* variable layout (oracle/params.py, a checkpoint, params_init.init_pwcnet)."""
        self.store.load(params)
        self._dirty = True

    def export_params(self):
        """Every variable, and with ema_decay its moving average under its ema_name."""
        return self.store.export_all()

    def averaged(self):
        """Context manager: inside it the network runs on its moving average and export_params() holds it under the plain names too; the
        live weights come back on exit (engine.averaged_weights).  Without averaging, nothing changes."""
        return averaged_weights(self, [self.store] if self.store.shadow is not None else [])

    def set_lr(self, lr):
        """The learning rate of the following optimiser steps (a device value: captured CUDA graphs read it too)."""
        self.lr.fill_(float(lr))

    # ------------------------------------------------------------------------------------------------ inputs
    def _batch(self, img1, img2, flow):
        if flow is None and self.loss != 'unsupervised':
            raise ValueError('the %s loss needs the ground-truth flow of the batch' % self.loss)
        return (img1, img2) if flow is None else (img1, img2, flow)

    def feed(self, img1, img2, flow=None):
        """Host -> device copy of one batch: frames [B,ih,iw,3] in [-0.5, 0.5] and their ground-truth flow [B,ih,iw,2] in PWC-Net's
        channel order (pinned host tensors copy asynchronously).  A batch that prefetch staged is handed over from its slot on the device.
        flow=None (unsupervised loss only): the frames alone; gt keeps what it held."""
        srcs = self._batch(img1, img2, flow)
        if self._uploads.take(img1, self.inputs[:len(srcs)]):
            return
        for dst, src in zip(self.inputs, srcs):
            dst.copy_(src, non_blocking=True)

    def prefetch(self, img1, img2, flow=None):
        """Starts the host -> device copy of an upcoming batch into a staging slot on the copy stream, so that it overlaps the kernels
        queued now; feed(img1, img2, flow) then hands it over on the device."""
        self._uploads.prefetch(self._batch(img1, img2, flow))

    def _copy_stream(self):
        if self._copy is None:
            self._copy = torch.cuda.Stream()
        return self._copy

    # ------------------------------------------------------------------------------------------------ execution
    def _ensure_packed(self):
        if self._dirty:
            self.pack.run()
            self._dirty = False

    def forward(self):
        """PWC-Net forward and the loss forward on the batch in img1 / img2 / gt (-> self.flow, self.sums), not augmented."""
        self._ensure_packed()
        self.copy_in.run()
        self.fwd.run()

    def train_step(self, allreduce=None, use_graph=False):
        """One step on the batch in img1 / img2 / gt: [augmentation], forward, loss, backward, [allreduce(flat gradient)], Adam + L2,
        re-pack.  use_graph replays two CUDA graphs (augmentation + forward + backward, optimiser + pack) around the all-reduce."""
        self._ensure_packed()
        if use_graph:
            fwd_bwd = self._capture('fwd_bwd', [self.aug, self.fwd, self.bwd])
            opt = self._capture('adam', [self.adam, self.pack], warm=False)
            fwd_bwd.replay()
            if allreduce is not None:
                allreduce(self.store.grad)
            opt.replay()
            return
        self.aug.run()
        self.fwd.run()
        self.bwd.run()
        if allreduce is not None:
            allreduce(self.store.grad)
        self.adam.run()
        self.pack.run()

    def _capture(self, key, plans, warm=True):
        return capture_plans(self.graphs, key, plans, warm=warm)

    def launches_per_step(self):
        return self.aug.count() + self.fwd.count() + self.bwd.count() + self.adam.count() + self.pack.count()

    # ------------------------------------------------------------------------------------------------ results
    def losses(self, reduce=None):
        """{flow_loss, flow_loss_l6 .. flow_loss_l2} of the last forward (device -> host read): level term = alpha_l / global batch *
        the level's sum over this rank's samples; flow_loss = their sum (the weight-decay term is applied by the optimiser, not
        included).  Unsupervised loss: {flow_loss, flow_loss_photo, flow_loss_smooth}, the census and the lambda_s-weighted smoothness
        terms of L over this rank's 2B directions, and their sum.  `reduce`: the SUM all-reduce of a data-parallel job."""
        t = self.sums
        if reduce is not None:
            t = t.clone()
            reduce(t)
        s = t.cpu().sum(0).tolist()
        if self.loss == 'unsupervised':
            norm = self.GB * self.H * self.W
            photo, smooth = s[0] / norm, self.smooth_weight * s[1] / norm
            return {'flow_loss': photo + smooth, 'flow_loss_photo': photo, 'flow_loss_smooth': smooth}
        terms = [a * v / self.GB for a, v in zip(self.alphas, s)]
        out = {'flow_loss_l%d' % l: v for l, v in zip(LEVELS, terms)}
        out['flow_loss'] = sum(terms)
        return out

    def direction_objective(self):
        """Unsupervised loss: P_n + lambda_s * Sm_n of each of the last forward's 2B directions (fp64 [2B] on the device; direction n < B
        is pair n, n >= B pair n - B swapped) -- the per-direction sums the validation adds up."""
        return (self.sums[:, 0] + self.smooth_weight * self.sums[:, 1]) / (self.H * self.W)

    def epe(self):
        """End-point error of the last forward's final flow (self.flow, the level-2 flow x4; its forward half for the unsupervised loss)
        against the ground truth it was trained or scored on (the augmented flow after an augmented train_step), on the ground truth's grid -> self.epe_sums, fp64 [B,4] on the device: per sample {sum e, 0, pixels, 0},
        e = ||pred - gt||_2 (cis_masked_epe with an all-ones mask; fixed-order sums).  When in_hw differs from H x W the prediction is first resized to in_hw with its vectors
        scaled to that grid (cis_crop_resize_flow_f32 over the whole frame)."""
        st = torch.cuda.current_stream().cuda_stream
        (ih, iw), H, W = self.in_hw, self.H, self.W
        if (ih, iw) != (H, W):
            for b in range(self.B):
                _lib.call('cis_crop_resize_flow_f32', self.flow[b].data_ptr(), H, W, 0, 0, H, W, self._pred_gt_grid[b].data_ptr(), ih, iw,
                          ih / H, iw / W, st)
        _lib.call('cis_masked_epe', self._pred_gt_grid.data_ptr(), self.batch[2].data_ptr(), self._ones.data_ptr(), self.B, ih * iw,
                  self._epe_scratch.data_ptr(), self.epe_sums.data_ptr(), st)
        return self.epe_sums
