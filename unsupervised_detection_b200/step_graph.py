"""Device-side step graph: everything adversarial_learner.py:72-258 puts in the TF graph, as static launch lists.

One `CISGraph` owns the parameters (flat fp32 master copies per scope), all activation buffers for a fixed
(batch, 384x640 -> HxW) geometry, and the launch lists: forward (PWC-Net -> resize -> generator -> mask (x) flow ->
3x recover -> Charbonnier losses), backward for the recover step, backward for the generator step, and clip + TF-Adam.
With masks='boxes' the same graph pretrains the recover net: random boxes (cis_box_masks) replace the generator, which is not built.
With flow_source='input' a supplied flow field replaces PWC-Net, for either mask source.
"""
import torch

from . import _lib
from .engine import Builder, ParamStore, Plan, Act
from .models.nets import GeneratorNet, RecoverNet
from .models.PWCNet.model_pwcnet import PWCNetBuilder

PWC_H, PWC_W = 384, 640   # data/davis2016_data_utils.py:87-88: frames are resized to 384x640 before PWC-Net


def box_sides(box_min, box_max, H, W):
    """Box side range of the recover-net pretraining from fractions of the image sides -> (lo_h, hi_h, lo_w, hi_w) in pixels:
    lo = max(1, floor(box_min * side)), hi = max(lo, floor(box_max * side)).  ValueError unless 0 < box_min <= box_max <= 1."""
    if not 0.0 < box_min <= box_max <= 1.0:
        raise ValueError('box fractions need 0 < box_min <= box_max <= 1, got box_min=%r box_max=%r' % (box_min, box_max))
    out = []
    for side in (H, W):
        lo = max(1, int(box_min * side))
        out += [lo, max(lo, int(box_max * side))]
    return tuple(out)


def capture_plans(graphs, key, plans, lane_key=0, warm=True):
    """The CUDA graph of `plans` cached in the dict `graphs` under `key`, captured on first use.  warm: run the plans once outside
    capture first (sets function attributes, lazy allocations) -- never for plans that change state (the optimiser step)."""
    g = graphs.get(key)
    if g is None:
        torch.cuda.synchronize()
        if warm:
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for pl in plans:
                    pl.run(lane_key=lane_key)
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for pl in plans:
                pl.run(lane_key=lane_key)
        graphs[key] = g
    return g


class UploadSlots(object):
    """Host -> device batch uploads on a copy stream for a graph whose batch fills the device buffers `like`: prefetch() copies an
    upcoming batch into one of two device staging slots, so that it overlaps the kernels queued now, and take() hands it over into the
    graph's inputs on the current stream.  Write-after-read: a slot is overwritten only once the main stream's last read of it has
    executed (the host can run steps ahead of the GPU).  copy_stream: callable -> the copy stream (made on first use)."""

    def __init__(self, like, copy_stream):
        self._like, self._copy_stream = tuple(like), copy_stream
        self._slots = None                  # two device staging slots, made on first prefetch
        self._slot = 0                      # the slot the last prefetch wrote
        self._read = [None, None]           # per slot: event after the main stream's last read of it (take)
        self._staged = None                 # (first host tensor, slot, copy-done event) of the last prefetched batch

    def upload(self, after, dst, srcs):
        """Host -> device copy of srcs into the device tensors dst on the copy stream, once event `after` (if any) has completed -> the
        event after the copy."""
        copy = self._copy_stream()
        if after is not None:
            copy.wait_event(after)
        with torch.cuda.stream(copy):
            for d, s in zip(dst, srcs):
                d.copy_(s, non_blocking=True)
            ready = torch.cuda.Event()
            ready.record(copy)
        return ready

    def prefetch(self, srcs):
        if self._slots is None:
            self._slots = [tuple(torch.empty_like(t) for t in self._like) for _ in range(2)]
        self._slot ^= 1
        self._staged = (srcs[0], self._slot, self.upload(self._read[self._slot], self._slots[self._slot], srcs))

    def take(self, key, dst):
        """When the last prefetch staged the batch whose first host tensor is `key`: copy it from its slot into dst on the current stream
        -> True; else False (nothing done)."""
        st = self._staged
        if st is None or st[0] is not key:
            return False
        _, slot, ready = st
        cur = torch.cuda.current_stream()
        cur.wait_event(ready)
        for d, s in zip(dst, self._slots[slot]):
            d.copy_(s, non_blocking=True)
        self._read[slot] = torch.cuda.Event()
        self._read[slot].record(cur)
        self._staged = None
        return True

    def drop(self):
        """Forget the staged batch: take() then hands nothing over until the next prefetch."""
        self._staged = None


class CISGraph(object):
    def __init__(self, img_height, img_width, batch, device='cuda', global_batch=None, flow_normalizer=80.0, cbn=0.5, epsilon=75.0,
                 beta1=0.9, with_pwc=True, train=True, pwc_hw=(PWC_H, PWC_W), seed=8964, pwc_options=None, masks=None, box=None,
                 sample_offset=0, flow_source='pwc'):
        """pwc_options: PWC-Net options (the reference's option keys; None = model_pwcnet._DEFAULT_PWCNET_TEST_OPTIONS).
        masks: 'generator' (the adversarial graph; None means it on PWC-Net's flow) or 'boxes' (pretraining of the recover net): one
        random box per sample, drawn on the device by cis_box_masks, replaces the generator's mask; the generator is neither run nor trained and only the recover step
        exists.  box = (lo_h, hi_h, lo_w, hi_w) box sides in pixels (None = box_sides(0.1, 0.5, H, W)); sample_offset = global index of
        this rank's first sample (rank * batch under data parallelism), so that every sample of the global batch gets its own box.
        with_pwc=False: no 384x640 inputs at all; image and flow are written at HxW directly (no stage, no pipelined schedule).
        flow_source: where the flow at 384x640 comes from.  'pwc' (the default): PWC-Net run on the frame pair img1 / img2.  'input':
        a known flow field uploaded into flow_full next to img1, in PWC-Net's channel order and sign; no PWC-Net is built.  The flow
        then reaches the generator and the recover net through the same resize and 1/flow_normalizer as PWC-Net's output, every launch
        after take_stage is the 'pwc' graph's, and the stage, the pipelined schedule and the batch hand-over work on the pair
        (img1, flow_full) in place of (img1, img2).  Both mask sources and train=True / False accept it, named explicitly: supplied
        flow serves the recover-net pretraining (masks='boxes') as well as the adversarial graph (masks='generator'), and a graph that
        silently became the other one would train the wrong network.  with_pwc=False does not accept it."""
        if masks is None:
            if flow_source == 'input':
                raise ValueError("flow_source='input' needs the mask source named: masks='generator' or masks='boxes'")
            masks = 'generator'
        _lib.load()
        if masks not in ('generator', 'boxes'):
            raise ValueError("masks must be 'generator' or 'boxes', got %r" % (masks,))
        if flow_source not in ('pwc', 'input'):
            raise ValueError("flow_source must be 'pwc' or 'input', got %r" % (flow_source,))
        if flow_source == 'input' and not with_pwc:
            raise ValueError("flow_source='input' needs the 384x640 inputs (with_pwc=True)")
        self.masks, self.flow_source = masks, flow_source
        boxes = masks == 'boxes'
        # Two attributes, two meanings: self.staged = the graph takes 384x640 uploads (self.inputs) that fwd.ops[:_pwc_ops] resizes into
        # the stage (the pipelined schedule needs this); self.with_pwc = PWC-Net is built (pwc_store, pack_pwc).  flow_source='input'
        # is staged without PWC-Net.
        staged = with_pwc
        with_pwc = with_pwc and flow_source == 'pwc'
        self.staged = staged
        self.box = tuple(box) if box is not None else box_sides(0.1, 0.5, img_height, img_width)
        self.sample_offset = sample_offset
        lo_h, hi_h, lo_w, hi_w = self.box
        if boxes and not (1 <= lo_h <= hi_h <= img_height and 1 <= lo_w <= hi_w <= img_width and sample_offset >= 0):
            raise ValueError('box sides %r need 1 <= lo <= hi <= the image side (%dx%d)' % (self.box, img_height, img_width))
        self.H, self.W, self.B = img_height, img_width, batch
        self.GB = global_batch or batch
        self.dev = device
        self.cbn, self.eps_rr, self.flow_norm, self.beta1 = cbn, epsilon, flow_normalizer, beta1
        self.with_pwc, self.train = with_pwc, train
        self.seed = seed
        f32 = lambda *s: torch.zeros(*s, dtype=torch.float32, device=device)
        B, H, W = batch, img_height, img_width
        # ---- parameter stores (scopes of adversarial_learner.py:211-214 and model_pwcnet.py)
        self.gen_store, self.rec_store, self.pwc_store = ParamStore(device), ParamStore(device), ParamStore(device)
        self.gen = GeneratorNet(self.gen_store)
        self.rec = RecoverNet(self.rec_store)
        self.gen_store.finalize(True)
        self.rec_store.finalize(True)
        if with_pwc:
            self.pwc = PWCNetBuilder(self.pwc_store, options=pwc_options)
            self.pwc_store.finalize(False)
        self.step_state = torch.zeros(1, dtype=torch.int64, device=device)   # shared Adam beta-power step (App. A.14)
        self.avg_abs = f32(1)
        # ---- static buffers
        bld = Builder(device)
        self.bld = bld
        P = bld.fwd
        self.img2 = None
        if with_pwc:
            ph, pw = pwc_hw
            self.img1, self.img2 = f32(B, ph, pw, 3), f32(B, ph, pw, 3)
            self.flow_full = f32(B, ph, pw, 2)
            i1 = Act(B, ph, pw, 3, device, name='img1_8')
            i2 = Act(B, ph, pw, 3, device, name='img2_8')
            npx = B * ph * pw
            P.add('cis_pack_f32_to_bf16', self.img1.data_ptr(), npx, 3, 0.5, i1.ptr, 8, 0)     # adapt_x: img + 0.5
            P.add('cis_pack_f32_to_bf16', self.img2.data_ptr(), npx, 3, 0.5, i2.ptr, 8, 0)
            self.pwc.build(bld, i1, i2, self.flow_full)
        elif staged:
            ph, pw = pwc_hw
            self.img1, self.flow_full = f32(B, ph, pw, 3), f32(B, ph, pw, 2)
        # the two device buffers one batch upload writes (feed, prefetch, feed_next): the frame pair, or frame 1 and its flow
        self.inputs = (self.img1, self.img2 if with_pwc else self.flow_full) if staged else None
        self.image = f32(B, H, W, 3)
        self.flow = f32(B, H, W, 2)
        self._pwc_ops = 0
        if staged:
            # adversarial_learner.py:87-97: legacy bilinear to (H,W); flow / flow_normalizer.  The frozen flow network writes its
            # results to STAGE buffers; the two small device copies below hand them to the trainable part.  That split is what lets
            # train_step(pipeline=True) run PWC-Net for the NEXT batch on a second stream while this batch trains (the flow network
            # has no dependency on the parameters being trained).  With flow_source='input' the prefix is these two resizes alone.
            self.image_st, self.flow_st = f32(B, H, W, 3), f32(B, H, W, 2)
            P.add('cis_resize_bilinear_f32', self.img1.data_ptr(), B, ph, pw, 3, self.image_st.data_ptr(), H, W, 1.0)
            P.add('cis_resize_bilinear_f32', self.flow_full.data_ptr(), B, ph, pw, 2, self.flow_st.data_ptr(), H, W, 1.0 / flow_normalizer)
            self._pwc_ops = len(P.ops)                  # fwd.ops[:_pwc_ops] = everything that depends only on the frame pair
            P.add_py(self._take_stage, 'take_stage')
        if not boxes:
            self.stats = torch.zeros(B, 4, dtype=torch.float64, device=device)
            self.gen_in = Act(B, H, W, 5, device, name='gen_in')
        self.img8 = Act(B, H, W, 3, device, name='img8')
        hw = H * W
        if not boxes:
            P.zero(self.stats)
            P.add('cis_flow_stats', self.flow.data_ptr(), B, hw, self.stats.data_ptr())                       # flow_utils.py:10
            P.add('cis_pack_generator_input', self.image.data_ptr(), self.flow.data_ptr(), self.stats.data_ptr(), B, hw, self.gen_in.ptr)
        P.add('cis_pack_f32_to_bf16', self.image.data_ptr(), B * hw, 3, 0.0, self.img8.ptr, 8, 0)
        self.mask = f32(B, H, W, 1)
        # held-out inpainting error of a boxes graph (masked_epe): per-sample sums and the kernel's block partials
        self.epe_sums = torch.zeros(B, 4, dtype=torch.float64, device=device) if boxes else None
        self._epe_scratch = torch.zeros(B * 256, dtype=torch.float64, device=device) if boxes else None
        if boxes:
            # The boxes depend on the Adam step counter, so this launch belongs to the main-lane part of the forward, after take_stage:
            # fwd.ops[:_pwc_ops] runs on the side stream in the pipelined schedule, concurrently with the previous step's Adam update.
            P.add('cis_box_masks', self.mask.data_ptr(), B, H, W, *self.box, sample_offset, self.step_state.data_ptr(), seed)
        bld.lane = 1
        i0 = len(P.ops)
        self.rec.build_a_encoder(bld, self.img8)        # side stream, overlaps the generator
        i1 = len(P.ops)
        bld.lane = 0
        if not boxes:
            self.gen.build(bld, self.gen_in, self.mask)
        mask_ops = P.ops[:i0] + P.ops[i1:]              # the forward ops that produce the masks (no recover net, no losses)
        # mask (x) flow -> recover inputs for the 3 calls (adversarial_learner.py:107-131)
        self.rec_in = Act(3 * B, H, W, 4, device, name='rec_in', dep=frozenset() if boxes else {'G'})
        if not boxes:
            self.rec_in.gen_rows = 2 * B
        P.add('cis_mask_apply', self.flow.data_ptr(), self.mask.data_ptr(), B, hw, self.rec_in.ptr)
        self.dmask = f32(B, H, W)
        logits = None if boxes else self.gen.logits

        def mask_bwd(bp, mode):
            if mode != 'G':
                return
            g = self.rec_in.get_grad()
            assert self.rec_in.grad_written.get('G'), 'recover backward did not reach the mask inputs'
            lg = logits.get_grad()
            bp.add('cis_mask_bwd', self.flow.data_ptr(), self.mask.data_ptr(), self.dmask.data_ptr(), g.ptr, B, hw, lg.ptr)
            logits.grad_written['G'] = True
        if not boxes:
            bld.tape.append(mask_bwd)
        h1, w1 = -(-H // 2), -(-W // 2)
        self.h1, self.w1 = h1, w1
        self.flow1 = f32(3 * B, h1, w1, 2)
        P.join()
        self.rec.build(bld, self.img8, self.rec_in, self.flow1)
        # ---- losses (adversarial_learner.py:141-204)
        self.sums = torch.zeros(B, 5, dtype=torch.float64, device=device)
        self.scalars = f32(8)
        self.coef = f32(B, 4)
        self.pred = f32(3 * B, H, W, 2)
        P.zero(self.sums)
        P.add('cis_cis_loss_fwd', self.flow.data_ptr(), self.mask.data_ptr(), self.flow1.data_ptr(), B, H, W, h1, w1, cbn,
              self.sums.data_ptr(), self.pred.data_ptr())
        P.add('cis_cis_loss_reduce', self.sums.data_ptr(), B, self.GB, hw, epsilon, self.scalars.data_ptr(), self.coef.data_ptr())
        self.fwd = P
        # ---- weight packing plans
        self.pack_pwc = Plan('pack_pwc')
        if with_pwc:
            for L in self.pwc.all_layers():
                L.plan_pack(self.pack_pwc)
        self.bwd = {}
        self.adam = {}
        if train:
            self.dpred = f32(3 * B, H, W, 2)
            for mode, which in (('R', 0),) if boxes else (('R', 0), ('G', 1)):
                nb = 3 * B if mode == 'R' else 2 * B
                head = Plan('loss_bwd_' + mode)
                head.add('cis_cis_loss_bwd', self.flow.data_ptr(), self.mask.data_ptr(), self.flow1.data_ptr(), self.coef.data_ptr(),
                         self.scalars.data_ptr(), B, H, W, h1, w1, cbn, which, self.dpred.data_ptr(), self.dmask.data_ptr())
                fg = self.rec.flow1.get_grad()
                head.add('cis_resize_f32_bwd_to_bf16', self.dpred.data_ptr(), nb, H, W, 2, h1, w1, fg.ptr, fg.pitch)
                store = self.store(mode)
                layers = self.rec.all_layers() if mode == 'R' else self.gen.all_layers()
                # nothing to zero: every real entry of the flat gradient buffer is overwritten by cis_unpack_wgrad / cis_bn_chain each
                # step, and its padding slots are never written (they stay at their initial 0, also through the all-reduce)
                self.bwd[mode] = bld.backward_plan(mode, head, [self.rec.flow1], layers)
                ad = Plan('adam_' + mode)
                if mode == 'G':
                    # can_change branch of train_op (loss_utils.py:18-26)
                    self.seg = torch.tensor([v for pr in store.seg_pairs for v in pr], dtype=torch.int64, device=device)
                    ad.zero(self.avg_abs)
                    ad.add('cis_grad_avg_abs', store.grad.data_ptr(), self.seg.data_ptr(), len(store.seg_pairs), self.avg_abs.data_ptr())
                ad.add('cis_clip_adam', store.flat.data_ptr(), store.m.data_ptr(), store.v.data_ptr(), store.grad.data_ptr(), store.size, 1.0,
                       0.2, 1e-4, beta1, 0.999, 1e-8, self.step_state.data_ptr(), self.avg_abs.data_ptr(), 1 if mode == 'G' else 0, seed)
                self.adam[mode] = ad
        # packing of the trainable nets (forward + data-gradient orientation), after backward planning decided what is needed
        self.pack_gen, self.pack_rec = Plan('pack_gen'), Plan('pack_rec')
        for L in self.gen.all_layers() if not boxes else ():    # box masks: the generator's parameters exist but nothing reads them
            L.plan_pack(self.pack_gen, dgrad=train)
        for L in self.rec.all_layers():
            L.plan_pack(self.pack_rec, dgrad=train)
        self.pack_gen, self.pack_rec, self.pack_pwc = (pl.batch_param_ops(device) for pl in (self.pack_gen, self.pack_rec, self.pack_pwc))
        self._pwc_packed = False
        self._dirty = True      # packed bf16 operands out of date w.r.t. the fp32 master weights
        self._mask_plan = self._sub_plan('fwd_masks', mask_ops)
        # the two parts of the forward in the pipelined step: the flow network (side stream) and everything after take_stage
        self._pipe_pwc = self._sub_plan('fwd_pwc', self.fwd.ops[:self._pwc_ops])
        self._pipe_rest = self._sub_plan('fwd_rest', self.fwd.ops[self._pwc_ops + 1:])
        # ---- device-only state, made on first use (a CISGraph is also built with device='cpu' to inspect its plans)
        self.graphs = {}                    # CUDA graphs by key (_capture_plans)
        self._side = self._copy = None      # streams of the pipelined flow-network branch and of batch uploads (_streams)
        self._uploads = UploadSlots(self.inputs or (), lambda: self._streams()[1])     # copy-stream uploads of (img1, img2)
        self._pipe_done = None              # event: the last pipelined step's flow-network branch has filled the stage
        self._pipe_free = None              # event: prime_pipeline has finished reading img1 / img2
        # Which frame pair is where.  A frame pair is named by its host img1 tensor when feed_next uploaded it, and by the device
        # buffer img1 when it was written there in any other way (feed, a direct copy).
        self.inputs_for = self.img1 if staged else None     # the frame pair in img1 / img2
        self.stage_for = None               # the frame pair whose flow the stage holds for the next pipelined step; None: stale

    # ------------------------------------------------------------------------------------------------ parameters
    def load_params(self, params):
        """params: dict name -> tensor with the reference's variable layout (see oracle/params.py for the names)."""
        self.gen_store.load(params)
        self.rec_store.load(params)
        self._dirty = True
        if self.with_pwc:
            self.pwc_store.load(params)
            self._pwc_packed = False

    def export_params(self):
        out = {}
        out.update(self.gen_store.export())
        out.update(self.rec_store.export())
        if self.with_pwc:
            out.update(self.pwc_store.export())
        return out

    def param_count(self):
        return self.gen_store.real_count() + self.rec_store.real_count() + (self.pwc_store.real_count() if self.with_pwc else 0)

    # ------------------------------------------------------------------------------------------------ execution
    def _ensure_packed(self):
        if self.with_pwc and not self._pwc_packed:
            self.pack_pwc.run()
            self._pwc_packed = True
        if self._dirty:
            self.pack_gen.run()
            self.pack_rec.run()
            self._dirty = False

    def store(self, mode):
        """The parameter store of the network that train step `mode` updates: 'R' the recover net, 'G' the generator."""
        return self.rec_store if mode == 'R' else self.gen_store

    def _pack_of(self, mode):
        return self.pack_rec if mode == 'R' else self.pack_gen

    def forward(self):
        self._ensure_packed()
        self.pipeline_drain()
        self.stage_for = None
        self.fwd.run()

    def forward_masks(self, use_graph=False):
        """Mask path only: [PWC-Net -> resize ->] flow normalisation -> generator -> self.mask (what test_generator*.py consume;
        the reference's multi-crop test graph, adversarial_learner.py:525-592, builds nothing else).  use_graph replays it as one
        CUDA graph."""
        self._ensure_packed()
        self.pipeline_drain()
        self.stage_for = None
        if use_graph:
            self._capture_plans('masks', [self._mask_plan]).replay()
        else:
            self._mask_plan.run()

    def forward_flow(self):
        """The frozen flow network alone on the frame pair in img1 / img2 -> self.flow_full [B,384,640,2] (PWC-Net's output, before the
        resize to HxW): what export_flow.py writes.  ValueError for a graph without PWC-Net."""
        if not self.with_pwc:
            raise ValueError('forward_flow needs a graph that runs PWC-Net')
        self._ensure_packed()
        self.pipeline_drain()
        self.stage_for = None
        self._pipe_pwc.run()

    def set_sample_offset(self, sample_offset):
        """Global index of the first sample for the box draws of the next eager forward() (a validation pass sets it per batch).  The
        offset is a launch argument, so CUDA graphs captured earlier would keep the old one: refused once one exists."""
        if self.masks != 'boxes' or self.graphs or sample_offset < 0:
            raise ValueError('set_sample_offset needs a boxes graph that has captured no CUDA graph and an offset >= 0')
        for plan in (self.fwd, self._mask_plan, self._pipe_rest):
            plan.ops = [op[:1] + (op[1][:8] + (sample_offset,) + op[1][9:],) + op[2:] if op[2] == 'cis_box_masks' else op for op in plan.ops]
        self.sample_offset = sample_offset

    def masked_epe(self):
        """Held-out inpainting error of the last forward of a boxes graph -> self.epe_sums, fp64 [B,4] on the device: per sample
        {sum m*e, sum (1-m)*e, sum m, sum (1-m)} with e = |pred - flow|_2 per HxW pixel, pred = the masked recover call (the first B
        rows of self.pred), m = the box mask.  e is in units of the normalised flow (times flow_normalizer: pixels of the 384x640
        grid).  Fixed-order reductions: bit-identical run to run."""
        _lib.call('cis_masked_epe', self.pred.data_ptr(), self.flow.data_ptr(), self.mask.data_ptr(), self.B, self.H * self.W,
                  self._epe_scratch.data_ptr(), self.epe_sums.data_ptr(), torch.cuda.current_stream().cuda_stream)
        return self.epe_sums

    def _take_stage(self):
        self.image.copy_(self.image_st, non_blocking=True)
        self.flow.copy_(self.flow_st, non_blocking=True)

    def launches_per_step(self, mode):
        return self.fwd.count() + self.bwd[mode].count() + self.adam[mode].count() + self._pack_of(mode).count()

    def train_step(self, mode, allreduce=None, use_graph=False, pipeline=False, inputs_ready=None):
        """One alternating step body (adversarial_learner.py:380-397): mode 'R' = train_recover_op, 'G' = train_generator_op.

        pipeline=True (CUDA graphs only): software pipeline over steps.  The step trains on the (image, flow) pair that the PREVIOUS
        call's side branch left in the stage buffers and, concurrently on a second stream, runs the frozen PWC-Net on the frame
        pair currently in self.img1 / self.img2 -- the NEXT batch -- for the next call.  `inputs_ready`: an event after which
        img1 / img2 hold that next batch (the host-to-device copy).  The first pipelined call primes the stage from img1 / img2.
        Results are identical to the sequential order; only the schedule changes."""
        if self.masks == 'boxes' and mode != 'R':
            raise ValueError("a masks='boxes' graph trains the recover net only (mode 'R'), got mode %r" % (mode,))
        self._ensure_packed()
        if use_graph and pipeline and self.staged:
            return self._train_step_pipelined(mode, allreduce, inputs_ready)
        if inputs_ready is not None:
            torch.cuda.current_stream().wait_event(inputs_ready)
        self.pipeline_drain()
        self.stage_for = None
        if use_graph:
            fwd_bwd = self._capture_plans('seq_fwd_bwd_' + mode, [self.fwd, self.bwd[mode]])
            adam = self._capture_plans('seq_adam_' + mode, [self.adam[mode], self._pack_of(mode)], warm=False)
            fwd_bwd.replay()
            if allreduce is not None:
                allreduce(self.store(mode).grad)
            adam.replay()
            return
        self.fwd.run()
        self.bwd[mode].run()
        if allreduce is not None:
            allreduce(self.store(mode).grad)
        self.adam[mode].run()
        self._pack_of(mode).run()      # only the updated network's bf16 operands are re-packed

    def _sub_plan(self, name, ops):
        sp = Plan(name)
        sp.ops = ops
        sp.keep = self.fwd.keep
        return sp

    def _capture_plans(self, key, plans, lane_key=0, warm=True):
        return capture_plans(self.graphs, key, plans, lane_key, warm)

    def _streams(self):
        """(side, copy): the stream of the pipelined flow-network branch and the stream of the host-to-device batch uploads."""
        if self._side is None:
            self._side, self._copy = torch.cuda.Stream(), torch.cuda.Stream()
        return self._side, self._copy

    def feed(self, img1, img2):
        """Host -> device copy of one batch of frame pairs [B,384,640,3] fp32 into img1 / img2 (pinned host tensors copy
        asynchronously).  A batch that prefetch staged is handed over from its staging slot on the device.  With
        flow_source='input' the second tensor is frame 1's flow [B,384,640,2] and goes to flow_full."""
        self.pipeline_drain()          # a pipelined flow-network branch may still be reading img1 / img2
        self.inputs_for = self.img1
        if self._uploads.take(img1, self.inputs):
            return
        self.inputs[0].copy_(img1, non_blocking=True)
        self.inputs[1].copy_(img2, non_blocking=True)

    def prefetch(self, img1, img2):
        """Starts the host -> device copy of an upcoming batch into a staging slot on the copy stream, so that it overlaps the kernels
        queued now; feed(img1, img2) then hands it over on the device."""
        self._uploads.prefetch((img1, img2))

    def feed_next(self, img1, img2):
        """Host -> device copy of the frame pair that the next pipelined train_step runs the flow network on, on the copy stream
        once the flow network has finished reading img1 / img2 -> the event to pass as train_step(inputs_ready=)."""
        ready = self._uploads.upload(self.pipeline_inputs_free(), self.inputs, (img1, img2))
        self.inputs_for = img1
        self._uploads.drop()
        return ready

    def prime_pipeline(self):
        """Run the frozen flow network (on the current stream) for the frame pair now in img1 / img2 so that the next
        train_step(pipeline=True) trains on it.  Needed before the first pipelined step and whenever the stream of batches restarts."""
        self._ensure_packed()
        self.pipeline_drain()
        self._capture_plans('pipe_pwc', [self._pipe_pwc], lane_key=1).replay()
        self._pipe_done = None
        self._pipe_free = torch.cuda.Event()
        self._pipe_free.record(torch.cuda.current_stream())
        self.stage_for = self.inputs_for

    def pipeline_inputs_free(self):
        """Event after which img1 / img2 may be overwritten with the next frame pair (the flow network last reading them is done)."""
        return self._pipe_done if self._pipe_done is not None else self._pipe_free

    def _train_step_pipelined(self, mode, allreduce, inputs_ready):
        main, side = torch.cuda.current_stream(), self._streams()[0]
        g_pwc = self._capture_plans('pipe_pwc', [self._pipe_pwc], lane_key=1)
        g_rest = self._capture_plans('pipe_rest_' + mode, [self._pipe_rest, self.bwd[mode]])
        g_adam = self._capture_plans('pipe_adam_' + mode, [self.adam[mode], self._pack_of(mode)], warm=False)
        if self.stage_for is None:
            # prime: the stage must hold the flow of the batch this call trains on (= what img1 / img2 hold right now)
            if inputs_ready is not None:
                main.wait_event(inputs_ready)
            self.prime_pipeline()
        if self._pipe_done is not None:
            main.wait_event(self._pipe_done)         # the previous call's side branch filled the stage
        self._take_stage()
        taken = torch.cuda.Event()
        taken.record(main)
        side.wait_event(taken)                       # stage and level buffers are free again
        if inputs_ready is not None:
            side.wait_event(inputs_ready)
        with torch.cuda.stream(side):
            g_pwc.replay()                           # PWC-Net on the NEXT batch, concurrent with everything below
            self._pipe_done = torch.cuda.Event()
            self._pipe_done.record(side)
        self.stage_for = self.inputs_for
        g_rest.replay()
        if allreduce is not None:
            allreduce(self.store(mode).grad)
        g_adam.replay()

    def pipeline_drain(self):
        """Join the side branch (call before reading PWC-Net outputs or re-feeding img1 / img2 outside train_step)."""
        if self._pipe_done is not None:
            torch.cuda.current_stream().wait_event(self._pipe_done)

    def losses(self, full=False, reduce=None):
        """The `losses` dict of adversarial_learner.py:196-204 (device -> host read).  full=True adds the four first-sample
        diagnostics (:201-204) taken from the per-sample Charbonnier sums {rec, rec_c, prior, den, den_c}.  `reduce`: the SUM
        all-reduce of a data-parallel job -- the local scalars are this rank's share of the global-batch losses."""
        if reduce is not None:
            t = self.scalars[:4].clone()
            reduce(t)
            s = t.tolist()
        else:
            s = self.scalars.tolist()
        out = dict(generator=s[0], recover=s[1], red_rate=s[2], red_rate_compl=s[3])
        if full:
            r = self.sums[0].tolist()
            out.update(reconstruction_loss=r[0], reconstruction_compl_loss=r[1], denominator_red_rate=r[3] + self.eps_rr,
                       denominator_red_rate_compl=r[4] + self.eps_rr)
        return out
