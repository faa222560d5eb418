"""Function-level surface of the reference on top of the launch-list engine (SURVEY 8b: `generator_net`, `recover_net`,
`charbonnier_loss`, `train_op`, `cost_volume`, `dense_image_warp`, `ModelPWCNet.predict_from_img_pairs` keep their names and NHWC
argument order; TF-only arguments -- scope / reuse / name / training -- are accepted, `scope` selects the parameter-name prefix).

The reference functions create TF graph nodes; here each call runs the corresponding sub-graph of libcis_b200 kernels on `cuda`
tensors and returns a device tensor.  Static launch plans are cached per input shape; parameters come from the `params` argument or
from the registry filled by `set_parameters()` (dict name -> tensor, names as in oracle/params.py / a loaded checkpoint).
PyTorch is used for memory and the small amount of buffer plumbing only; there is no CPU fallback: without the CUDA library (or on CPU
tensors) the calls raise.

The layer primitives of models/utils/convolution_utils.py (resize, resize_bilinear, resize_nearest_neighbor, gen_conv, gen_deconv, conv,
deconv) and flow_utils.preprocess_flow_batch are here too, for building variants of the two networks: each conv call is one ConvLayer
of the engine in a runner of its own (_LayerRunner), the resizes and the flow standardisation are stand-alone fp32 kernels.

Gradients: generator_net, recover_net, ModelPWCNet.predict_from_img_pairs, charbonnier_loss, cost_volume(_r), dense_image_warp and the
layer primitives are torch.autograd Functions (first order only) when an input or one of the parameter tensors the call reads requires
grad; the parameters then receive gradients under their variable names.  The backward runs the engine's backward kernels (data / weight gradients, BN chain
rule, resize transposes, the PWC-Net warp + cost-volume and transposed-conv backward) and the backward kernels of the three stand-alone
ops.  A call that needs no gradient runs exactly the forward-only path.  train_op is an optimiser update and has nothing to differentiate.
The training step (step_graph.py) still treats PWC-Net as frozen, as the reference does.

The sub-graphs reuse the builders that the step graph is made of; tests/test_functional_api_gpu.py and
tests/test_functional_grad_gpu.py check them against the oracle on the GPU, tests/test_functional_api_cpu.py and
tests/test_functional_grad_cpu.py check the plumbing and the plans without one.
"""
import torch
from torch.autograd.function import once_differentiable

from .. import _lib
from ..engine import Act, Builder, ConvLayer, ParamStore, Plan, ru
from .nets import GeneratorNet, RecoverNet

_PARAMS = {}
_RUNNERS = {}
_POOLS = {}      # runner key -> free runner instances of gradient-carrying calls


def set_parameters(params):
    """Register parameters (name -> tensor) for the functional calls; later registrations override earlier ones."""
    _PARAMS.update(params)
    for r in _RUNNERS.values():
        r.dirty = True


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _check_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError('the functional API runs the CUDA library on device tensors; got a %s tensor (no CPU fallback)' % t.device)


def _scope_name(scope, default):
    return (scope or default).rstrip('/') or default


class _NetRunner(object):
    """One cached static plan: parameter store + packed operands + input/output buffers for a fixed shape.  `bwd` is the backward plan
    (built by ensure_backward for the runners of gradient-carrying calls only); `runs` counts forward runs.  SEED names the fp32 buffer the
    backward plan reads the output gradient from, INPUT_GRADS the fp32 buffers it leaves the input gradients in (in argument order)."""

    MODE = None
    SEED = None
    INPUT_GRADS = ()

    def __init__(self, device):
        self.device = device
        self.store = ParamStore(device)
        self.bld = Builder(device)
        self.pack = Plan('pack')
        self.dirty = True
        self._loaded = None
        self.bwd = None
        self.runs = 0

    def finish(self, layers):
        self.layers = layers
        for L in layers:
            L.plan_pack(self.pack)

    def load(self, params):
        src = params if params is not None else _PARAMS
        if self.dirty or self._loaded is not src:
            self.store.load(src)
            self.pack.run()
            self.dirty, self._loaded = False, src

    def reload(self, params):
        """Unconditional load + pack (a gradient-carrying call: the parameter tensors may have been updated in place since)."""
        self.store.load(params)
        self.pack.run()
        self.dirty, self._loaded = False, None

    def param_names(self):
        return [e[0] for e in self.store.entries]

    def ensure_backward(self):
        """Backward plan: seed (`_plan_seed`) -> the builder's reverse tape -> fixed-order weight-gradient reduction + BN chain rule
        (one cis_param_multi launch per kind) -> input gradients out of the bf16 input Acts (`_plan_inputs`).  The pack plan is rebuilt
        with the data-gradient operands the tape needs."""
        if self.bwd is not None:
            return
        self.store.grad = torch.zeros_like(self.store.flat)
        seed, seeds = self._plan_seed()
        body = self.bld.build_backward(self.MODE, seeds)
        fin = Plan('fin')
        for L in self.layers:
            L.plan_finalize(fin, self.MODE)
        full = Plan('bwd_' + self.MODE)
        full.extend(seed)
        full.extend(body)
        full.join()            # weight-gradient lane -> main lane before the packed gradients are unpacked
        full.extend(fin.batch_param_ops(self.device))
        full.extend(self._plan_inputs())
        self.bwd = full
        self.pack = Plan('pack')
        for L in self.layers:
            L.plan_pack(self.pack, dgrad=True)
        self.dirty = True

    def param_grads(self):
        return [self.store.view(n, 'grad').clone() for n in self.param_names()]


class _GeneratorRunner(_NetRunner):
    MODE, SEED, INPUT_GRADS = 'G', 'dmask', ('dimage', 'dflow')

    def __init__(self, B, H, W, device, scope):
        _NetRunner.__init__(self, device)
        self.net = GeneratorNet(self.store, scope)
        self.store.finalize(False)
        f32 = self.bld.f32
        self.B, self.H, self.W = B, H, W
        self.image, self.flow, self.mask = f32(B, H, W, 3), f32(B, H, W, 2), f32(B, H, W, 1)
        # generator_net receives the ALREADY normalised flow (adversarial_learner.py:100-105); cis_pack_generator_input normalises with
        # the statistics it is given, so feed it mean 0 / variance 1: {sum, sum, sum of squares, sum of squares} = {0, 0, hw, hw}
        self.stats = torch.tensor([[0.0, 0.0, float(H * W), float(H * W)]] * B, dtype=torch.float64, device=device)
        # dependency 'G': a backward plan emits conv1's data gradient into gen_in.grad (image and flow gradients)
        self.gen_in = self.bld.new_act(B, H, W, 5, name='gen_in', dep={'G'})
        self.bld.fwd.add('cis_pack_generator_input', self.image.data_ptr(), self.flow.data_ptr(), self.stats.data_ptr(), B, H * W, self.gen_in.ptr)
        self.net.build(self.bld, self.gen_in, self.mask)
        self.finish(self.net.all_layers())

    def run(self, images, flows):
        self.image.copy_(images)
        self.flow.copy_(flows)
        self.bld.fwd.run()
        self.runs += 1
        return self.mask.clone()

    def __call__(self, images, flows, params):
        self.load(params)
        return self.run(images, flows)

    def _plan_seed(self):
        f32 = self.bld.f32
        B, H, W = self.B, self.H, self.W
        self.dmask, self.dimage, self.dflow = f32(B, H, W, 1), f32(B, H, W, 3), f32(B, H, W, 2)
        lg = self.net.logits.get_grad()
        seed = Plan('seed_G')
        # mask = sigmoid((l0 - l1) / 10) fused into conv17's epilogue: dmask -> dlogits (no recover-input chain)
        seed.add('cis_mask_bwd', None, self.mask.data_ptr(), self.dmask.data_ptr(), None, B, H * W, lg.ptr)
        return seed, [self.net.logits]

    def _plan_inputs(self):
        assert self.gen_in.grad_written.get('G'), "generator backward did not reach conv1's data gradient"
        g, npix = self.gen_in.get_grad(), self.B * self.H * self.W
        P = Plan('inputs_G')
        P.add('cis_cast_bf16_to_f32', g.ptr, npix, g.pitch, 0, 3, self.dimage.data_ptr())    # image: channels 0-2
        P.add('cis_cast_bf16_to_f32', g.ptr, npix, g.pitch, 3, 2, self.dflow.data_ptr())     # normalised flow: channels 3-4
        return P


class _RecoverRunner(_NetRunner):
    MODE, SEED, INPUT_GRADS = 'R', 'dpred', ('dimage', 'dflow', 'dmask')

    def __init__(self, B, H, W, device, scope, f):
        _NetRunner.__init__(self, device)
        self.net = RecoverNet(self.store, scope, f)
        self.store.finalize(False)
        f32 = self.bld.f32
        self.B, self.H, self.W = B, H, W
        self.h1, self.w1 = -(-H // 2), -(-W // 2)
        self.image, self.aug = f32(B, H, W, 3), f32(B, H, W, 4)
        self.flow1, self.pred = f32(B, self.h1, self.w1, 2), f32(B, H, W, 2)
        # dependency 'R': a backward plan emits aconv1's / bconv1's data gradients into the two input Acts
        self.img8 = self.bld.new_act(B, H, W, 3, name='img8', dep={'R'})
        self.flow_in = self.bld.new_act(B, H, W, 4, name='rec_in', dep={'R'})
        P = self.bld.fwd
        P.add('cis_pack_f32_to_bf16', self.image.data_ptr(), B * H * W, 3, 0.0, self.img8.ptr, 8, 0)
        P.add('cis_pack_f32_to_bf16', self.aug.data_ptr(), B * H * W, 4, 0.0, self.flow_in.ptr, 8, 0)
        self.net.build(self.bld, self.img8, self.flow_in, self.flow1, ncalls=1)
        P.join()
        P.add('cis_resize_bilinear_f32', self.flow1.data_ptr(), B, self.h1, self.w1, 2, self.pred.data_ptr(), H, W, 1.0)   # nets.py:108
        self.finish(self.net.all_layers())

    def run(self, img1, flow_masked, mask):
        self.image.copy_(img1)
        # input augmentation of nets.py:50-53: [flow_masked, ones, 1 - mask]
        self.aug[..., 0:2].copy_(flow_masked)
        self.aug[..., 2:3].fill_(1.0)
        self.aug[..., 3:4].copy_(1.0 - mask)
        self.bld.fwd.run()
        self.runs += 1
        return self.pred.clone()

    def __call__(self, img1, flow_masked, mask, params):
        self.load(params)
        return self.run(img1, flow_masked, mask)

    def _plan_seed(self):
        f32 = self.bld.f32
        B, H, W = self.B, self.H, self.W
        self.dpred, self.dimage, self.dflow, self.dmask = f32(B, H, W, 2), f32(B, H, W, 3), f32(B, H, W, 2), f32(B, H, W, 1)
        fg = self.net.flow1.get_grad()
        seed = Plan('seed_R')
        # transpose of the final legacy-bilinear x2 (nets.py:108), as in the step graph's loss head
        seed.add('cis_resize_f32_bwd_to_bf16', self.dpred.data_ptr(), B, H, W, 2, self.h1, self.w1, fg.ptr, fg.pitch)
        return seed, [self.net.flow1]

    def _plan_inputs(self):
        assert self.img8.grad_written.get('R') and self.flow_in.grad_written.get('R'), 'recover backward did not reach its inputs'
        gi, gf, npix = self.img8.get_grad(), self.flow_in.get_grad(), self.B * self.H * self.W
        P = Plan('inputs_R')
        P.add('cis_cast_bf16_to_f32', gi.ptr, npix, gi.pitch, 0, 3, self.dimage.data_ptr())
        P.add('cis_cast_bf16_to_f32', gf.ptr, npix, gf.pitch, 0, 2, self.dflow.data_ptr())                  # flow_masked: channels 0-1
        P.add('cis_cast_bf16_to_f32_scaled', gf.ptr, npix, gf.pitch, 3, 1, -1.0, self.dmask.data_ptr())     # channel 3 = 1 - mask
        return P


class _PWCRunner(_NetRunner):
    """trainable=False: the forward-only plan of calls without gradients.  trainable=True: layers tagged 'P', backward recorded.
    options: the PWC-Net options (None = model_pwcnet._DEFAULT_PWCNET_TEST_OPTIONS)."""
    MODE, SEED, INPUT_GRADS = 'P', 'dflow_out', ('dimg1', 'dimg2')

    def __init__(self, B, H, W, device, name, trainable=False, options=None):
        from .PWCNet.model_pwcnet import PWCNetBuilder
        _NetRunner.__init__(self, device)
        self.net = PWCNetBuilder(self.store, name, trainable=trainable, options=options)
        self.store.finalize(False)
        f32 = self.bld.f32
        self.B, self.H, self.W = B, H, W
        self.img1, self.img2, self.flow = f32(B, H, W, 3), f32(B, H, W, 3), f32(B, H, W, 2)
        # dependency 'P': a backward plan emits conv1a's data gradients (both frames) into the two image Acts
        dep = {'P'} if trainable else frozenset()
        self.i1, self.i2 = self.bld.new_act(B, H, W, 3, name='img1_8', dep=dep), self.bld.new_act(B, H, W, 3, name='img2_8', dep=dep)
        P = self.bld.fwd
        P.add('cis_pack_f32_to_bf16', self.img1.data_ptr(), B * H * W, 3, 0.5, self.i1.ptr, 8, 0)      # adapt_x: images arrive in [-0.5, 0.5]
        P.add('cis_pack_f32_to_bf16', self.img2.data_ptr(), B * H * W, 3, 0.5, self.i2.ptr, 8, 0)
        self.net.build(self.bld, self.i1, self.i2, self.flow)
        self.finish(self.net.all_layers())

    def run(self, img1, img2):
        self.img1.copy_(img1)
        self.img2.copy_(img2)
        self.bld.fwd.run()
        self.runs += 1
        return self.flow.clone()

    def __call__(self, img1, img2, params):
        self.load(params)
        return self.run(img1, img2)

    def _plan_seed(self):
        from .PWCNet.model_pwcnet import FLOW_PRED_LVL
        f32 = self.bld.f32
        B, H, W = self.B, self.H, self.W
        self.dflow_out, self.dimg1, self.dimg2 = f32(B, H, W, 2), f32(B, H, W, 3), f32(B, H, W, 3)
        seed = Plan('seed_P')
        for g in self.net.level_grad.values():      # the DenseNet level gradients accumulate from zero
            seed.zero(g)
        fb = self.net.flows_bf[FLOW_PRED_LVL]
        fg, s = fb.get_grad(), 2 ** FLOW_PRED_LVL
        # transpose of the final legacy-bilinear x4 and its x4 scale (model_pwcnet.py:642-647) into the level-2 flow gradient
        seed.add('cis_resize_f32_bwd_to_bf16_scaled', self.dflow_out.data_ptr(), B, H, W, 2, H // s, W // s, fg.ptr, fg.pitch, float(s))
        return seed, [fb]

    def _plan_inputs(self):
        assert self.i1.grad_written.get('P') and self.i2.grad_written.get('P'), 'PWC-Net backward did not reach its inputs'
        npix = self.B * self.H * self.W
        P = Plan('inputs_P')
        for a, d in ((self.i1, self.dimg1), (self.i2, self.dimg2)):      # image + 0.5 (adapt_x): unit derivative
            g = a.get_grad()
            P.add('cis_cast_bf16_to_f32', g.ptr, npix, g.pitch, 0, 3, d.data_ptr())
        return P


class _LayerRunner(_NetRunner):
    """One layer primitive of convolution_utils.py on a fixed input shape: f32 -> bf16 pack of the input, an optional pre-op ('nn2x':
    NN x2 with align_corners, gen_deconv; 'bilinear': the legacy resize to `size`, deconv), then one ConvLayer -- bias, inference BN
    folded into the weights (gen_conv), fused activation -- that writes the bf16 Act its activation derivative reads and the fp32 output
    the call returns.  spec = (kind, k, cout, stride, rate, act, pre, size, name); kind 'gen' = gen_conv parameters
    <name>/kernel|bias|gamma|beta, 'conv' = <name>/weights|biases."""
    MODE, SEED, INPUT_GRADS = 'L', 'dout', ('dx',)

    def __init__(self, B, H, W, cin, spec, device):
        _NetRunner.__init__(self, device)
        kind, k, cout, stride, rate, act, pre, size, name = spec
        gen = kind == 'gen'
        self.layer = ConvLayer(self.store, name, k, cin, cout, stride, rate, act, 0.2, tag='L', bn=gen,
                               wname='kernel' if gen else 'weights', bname='bias' if gen else 'biases')
        self.store.finalize(False)
        f32 = self.bld.f32
        self.B, self.H, self.W, self.cin = B, H, W, cin
        # the input is staged in a buffer padded to the bf16 Act's 8-channel pitch, so one cast kernel packs it; padding stays zero
        self.x_pad = f32(B, H, W, ru(cin, 8))
        self.x = self.x_pad[..., :cin]
        # dependency 'L': the backward plan emits the conv's data gradient (through the pre-op) into x8.grad
        self.x8 = self.bld.new_act(B, H, W, cin, name='x8', dep={'L'})
        self.bld.fwd.add('cis_cast_f32_to_bf16', self.x_pad.data_ptr(), self.x_pad.numel(), self.x8.ptr)
        src = self.x8
        if pre == 'nn2x':
            src = self.bld.upsample_nn2x(src)
        elif pre == 'bilinear':
            src = self.bld.resize_bilinear(src, size[0], size[1])
        self.outf = f32(B, -(-src.H // stride), -(-src.W // stride), cout)
        self.out = self.bld.conv(self.layer, [src], outf=self.outf)
        self.finish([self.layer])

    def run(self, x):
        self.x.copy_(x)
        self.bld.fwd.run()
        self.runs += 1
        return self.outf.clone()

    def __call__(self, x, params):
        self.load(params)
        return self.run(x)

    def _plan_seed(self):
        f32 = self.bld.f32
        B, OH, OW, cout = self.outf.shape
        self.dout_pad = f32(B, OH, OW, ru(cout, 8))
        self.dout = self.dout_pad[..., :cout]
        self.dx = f32(self.B, self.H, self.W, self.cin)
        g = self.out.get_grad()
        seed = Plan('seed_L')
        seed.add('cis_cast_f32_to_bf16', self.dout_pad.data_ptr(), self.dout_pad.numel(), g.ptr)
        return seed, [self.out]

    def _plan_inputs(self):
        assert self.x8.grad_written.get('L'), "layer backward did not reach the input's data gradient"
        g = self.x8.get_grad()
        P = Plan('inputs_L')
        P.add('cis_cast_bf16_to_f32', g.ptr, self.B * self.H * self.W, g.pitch, 0, self.cin, self.dx.data_ptr())
        return P


def _runner(kind, key, make):
    k = (kind,) + key
    r = _RUNNERS.get(k)
    if r is None:
        _lib.load()
        r = _RUNNERS[k] = make()
    return r


class _Lease(object):
    """A runner instance taken from the per-shape free list by one gradient-carrying call.  Runners hold static activation buffers, so
    every call that is still waiting for its backward needs its own instance; the lease puts it back when the backward has run or when
    the call's autograd context is released (no backward will come)."""

    def __init__(self, free, runner):
        self.free, self.runner = free, runner
        self.run_id = None

    def take(self):
        r = self.runner
        if r is None:
            raise RuntimeError('this call has already run its backward (the functional API is first-order: no retain_graph / double backward)')
        if r.runs != self.run_id:
            raise RuntimeError('the runner of this call was re-run after its forward; its activations are gone')
        return r

    def release(self):
        r, self.runner = self.runner, None
        if r is not None:
            self.free.append(r)

    def __del__(self):
        self.release()


def _lease(kind, key, make):
    free = _POOLS.setdefault((kind,) + key, [])
    if free:
        r = free.pop()
    else:
        _lib.load()
        r = make()
        r.ensure_backward()
    return _Lease(free, r)


def _param_inputs(runner, params):
    """(names, tensors) of the parameters a call reads, in the runner's store order."""
    src = params if params is not None else _PARAMS
    names = runner.param_names()
    missing = [n for n in names if n not in src]
    if missing:
        raise KeyError('missing parameter ' + missing[0])
    return names, [src[n] for n in names]


def _needs_grad(tensors):
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors)


class _NetFn(torch.autograd.Function):
    """generator_net / recover_net / predict_from_img_pairs with their parameters as explicit inputs:
    apply(lease, names, n_in, *inputs, *parameters)."""

    @staticmethod
    def forward(ctx, lease, names, n_in, *args):
        r = lease.runner
        r.reload(dict(zip(names, args[n_in:])))
        out = r.run(*args[:n_in])
        lease.run_id = r.runs
        ctx.lease = lease
        ctx.like = [(t.device, t.dtype, t.shape) for t in args]
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, gout):
        r = ctx.lease.take()
        getattr(r, r.SEED).copy_(gout)
        r.bwd.run()
        grads = [getattr(r, n).clone() for n in r.INPUT_GRADS] + r.param_grads()
        ctx.lease.release()
        out = []
        for need, g, (dev, dt, shape) in zip(ctx.needs_input_grad[3:], grads, ctx.like):
            out.append(g.to(device=dev, dtype=dt).reshape(shape) if need else None)
        return (None, None, None) + tuple(out)


# ------------------------------------------------------------------------------------------------------------------ networks
def generator_net(images, flows, scope='MaskNet', reuse=None, training=True, params=None):
    """models/nets.py:4-42 -> generated mask [B,H,W,1] in (0,1).  images [B,H,W,3] in [-0.5,0.5], flows [B,H,W,2] normalised.
    Differentiable w.r.t. images, flows and every '<scope>/...' parameter (bf16 activations, fp32 gradients)."""
    _check_cuda(images, flows)
    B, H, W, _ = images.shape
    sc = _scope_name(scope, 'MaskNet')
    key = (B, H, W, str(images.device), sc)
    make = lambda: _GeneratorRunner(B, H, W, images.device, sc)
    r = _runner('gen', key, make)
    names, pvals = _param_inputs(r, params)
    if not _needs_grad([images, flows] + pvals):
        return r(images, flows, params)
    lease = _lease('gen', key, make)
    try:
        return _NetFn.apply(lease, names, 2, images, flows, *pvals)
    except BaseException:
        lease.release()
        raise


def recover_net(img1, flow_masked, mask, scope='FlownetS', reuse=None, f=0.25, training=True, params=None):
    """models/nets.py:45-110 -> recovered flow [B,H,W,2] at the input resolution.  Differentiable w.r.t. img1, flow_masked, mask and
    every '<scope>/...' parameter.  Every call that still waits for its backward holds its own runner instance, so a loss may call it
    several times (three times in adversarial_learner.py:112-131) before one backward."""
    _check_cuda(img1, flow_masked, mask)
    B, H, W, _ = img1.shape
    sc = _scope_name(scope, 'FlownetS')
    key = (B, H, W, str(img1.device), sc, f)
    make = lambda: _RecoverRunner(B, H, W, img1.device, sc, f)
    r = _runner('rec', key, make)
    names, pvals = _param_inputs(r, params)
    if not _needs_grad([img1, flow_masked, mask] + pvals):
        return r(img1, flow_masked, mask, params)
    lease = _lease('rec', key, make)
    try:
        return _NetFn.apply(lease, names, 3, img1, flow_masked, mask, *pvals)
    except BaseException:
        lease.release()
        raise


def predict_from_img_pairs(img1, img2, name='pwcnet', params=None, options=None):
    """ModelPWCNet.predict_from_img_pairs (model_pwcnet.py:39-76): forward flow img1 -> img2, [B,H,W,2] in pixels of the input size
    (H, W multiples of 64, 384x640 in the reference's pipeline).  Differentiable w.r.t. img1, img2 and every '<name>/...' parameter
    (kernels HWIO, transposed-conv kernels [kh,kw,Cout,Cin]; bf16 activations, fp32 gradients), for fine-tuning the flow network or
    gradients with respect to the frames.  The training step keeps PWC-Net frozen, as the reference does (adversarial_learner.py:211-234).
    options: the PWC-Net options (dense connections, context network, search range; None = the module default), part of the plan key."""
    from .PWCNet.model_pwcnet import normalize_options
    _check_cuda(img1, img2)
    B, H, W, _ = img1.shape
    if H % 64 or W % 64:
        raise ValueError('PWC-Net needs input sizes that are multiples of 64 (6 pyramid levels); got %dx%d' % (H, W))
    opts = normalize_options(options)
    key = (B, H, W, str(img1.device), name, opts)
    r = _runner('pwc', key, lambda: _PWCRunner(B, H, W, img1.device, name, options=opts))
    names, pvals = _param_inputs(r, params)
    if not _needs_grad([img1, img2] + pvals):
        return r(img1, img2, params)
    lease = _lease('pwc', key, lambda: _PWCRunner(B, H, W, img1.device, name, trainable=True, options=opts))
    try:
        return _NetFn.apply(lease, names, 2, img1, img2, *pvals)
    except BaseException:
        lease.release()
        raise


# -------------------------------------------------------------------------------------------------------------------- losses
def charbonnier_loss(gt_flows, pred_flows, masks, cbn=0.5):
    """models/utils/loss_utils.py:34-51 -> [B]: sum over H, W, C of ((gt - pred)^2 + 0.001^2)^cbn * mask."""
    _check_cuda(gt_flows, pred_flows, masks)
    B, H, W, C = gt_flows.shape
    mc = masks.shape[-1]
    if tuple(masks.shape[:3]) != (B, H, W) or mc not in (1, C) or tuple(pred_flows.shape) != (B, H, W, C):
        raise ValueError('charbonnier_loss: shapes %s / %s / %s' % (tuple(gt_flows.shape), tuple(pred_flows.shape), tuple(masks.shape)))
    if _needs_grad([gt_flows, pred_flows, masks]):
        return _CharbonnierFn.apply(gt_flows, pred_flows, masks, float(cbn))
    return _charbonnier_fwd(gt_flows, pred_flows, masks, cbn)[0]


def _charbonnier_fwd(gt_flows, pred_flows, masks, cbn):
    B, H, W, C = gt_flows.shape
    g, p, m = (t.contiguous().float() for t in (gt_flows, pred_flows, masks))
    sums = torch.zeros(B, dtype=torch.float64, device=g.device)
    _lib.call('cis_charbonnier_sum', g.data_ptr(), p.data_ptr(), m.data_ptr(), B, H * W, C, m.shape[-1], float(cbn), sums.data_ptr(), _stream())
    return sums.float(), (g, p, m)


def _ptr(t):
    return t.data_ptr() if t is not None else None


class _CharbonnierFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, gt_flows, pred_flows, masks, cbn):
        out, gpm = _charbonnier_fwd(gt_flows, pred_flows, masks, cbn)
        ctx.save_for_backward(*gpm)
        ctx.cbn = cbn
        ctx.dtypes = (gt_flows.dtype, pred_flows.dtype, masks.dtype)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, dsum):
        g, p, m = ctx.saved_tensors
        B, H, W, C = g.shape
        need = ctx.needs_input_grad
        dgt, dpred, dmask = (torch.empty_like(t) if n else None for t, n in zip((g, p, m), need[:3]))
        ds = dsum.contiguous().float()
        _lib.call('cis_charbonnier_bwd', g.data_ptr(), p.data_ptr(), m.data_ptr(), B, H * W, C, m.shape[-1], ctx.cbn, ds.data_ptr(),
                  _ptr(dpred), _ptr(dgt), _ptr(dmask), _stream())
        out = tuple(d.to(dt) if d is not None else None for d, dt in zip((dgt, dpred, dmask), ctx.dtypes))
        return out + (None,)


def train_op(params, grads, m, v, step_state, gradient_clip_value=0.1, can_change=False, learning_rate=1e-4, beta1=0.9, beta2=0.999,
             epsilon=1e-8, segments=None, seed=8964):
    """models/utils/loss_utils.py:12-32 + tf.train.AdamOptimizer.apply_gradients on FLAT fp32 device buffers (one per variable scope):
    clip to +-gradient_clip_value -- or, when `can_change` and the mean over variables of mean|g| is below 1e-5, replace the gradient by
    |U(-clip, clip)| noise -- then one TF-form Adam update.  `step_state`: int64 [1] shared step counter (the beta powers of
    adversarial_learner.py:216); `segments`: int64 [nvar, 2] = (start, end) of every variable in the flat buffer (needed for can_change)."""
    _check_cuda(params, grads, m, v, step_state)
    avg = torch.zeros(1, dtype=torch.float32, device=params.device)
    if can_change:
        if segments is None:
            raise ValueError('train_op(can_change=True) needs the variable segments of the flat gradient buffer')
        seg = segments.to(device=params.device, dtype=torch.int64).contiguous()
        _lib.call('cis_grad_avg_abs', grads.data_ptr(), seg.data_ptr(), seg.shape[0], avg.data_ptr(), _stream())
    _lib.call('cis_clip_adam', params.data_ptr(), m.data_ptr(), v.data_ptr(), grads.data_ptr(), params.numel(), 1.0, float(gradient_clip_value),
              float(learning_rate), float(beta1), float(beta2), float(epsilon), step_state.data_ptr(), avg.data_ptr(), 1 if can_change else 0,
              int(seed), _stream())
    return params


# ---------------------------------------------------------------------------------------------------------------- PWC-Net ops
def _to_act(x):
    """fp32 [B,h,w,C] -> bf16 NHWC buffer with the channel count padded to a multiple of 8 (the kernels' 16-byte pixel chunks)."""
    B, h, w, C = x.shape
    c8 = (C + 7) // 8 * 8
    buf = torch.zeros(B, h, w, c8, dtype=torch.bfloat16, device=x.device)
    buf[..., :C] = x.to(torch.bfloat16)
    return Act(B, h, w, C, x.device, buf=buf)


def cost_volume(c1, warp, search_range=4, name=None):
    """models/PWCNet/core_costvol.py:20-40 -> [B,h,w,81]: leaky_relu(mean_c c1 * shifted warp, 0.1), zero padded, dy outer, for the
    reference's default search_range = 4; features and result are bf16-rounded like in the pipeline.  Differentiable w.r.t. c1 and warp
    (gradients of the bf16-rounded features, fp32).  Other ranges raise NotImplementedError here; cost_volume_r takes ranges 1..4."""
    if search_range != 4:
        raise NotImplementedError('cost_volume: implements search_range=4 (model_pwcnet.py options); cost_volume_r(c1, warp, search_range) '
                                  'takes 1, 2, 3 and 4')
    return cost_volume_r(c1, warp, 4)


def cost_volume_r(c1, warp, search_range, name=None):
    """cost_volume for search_range 1..4 -> [B,h,w,(2r+1)^2] (model_pwcnet.py option 'search_range'): the same op, forward and gradient,
    on the fused kernels' range variants; range 4 runs exactly cost_volume."""
    _check_cuda(c1, warp)
    if isinstance(search_range, bool) or search_range not in (1, 2, 3, 4):
        raise NotImplementedError('cost_volume_r: the fused kernels implement search_range 1, 2, 3 and 4; got %r' % (search_range,))
    r = int(search_range)
    if _needs_grad([c1, warp]):
        return _CostVolumeFn.apply(c1, warp, r)
    return _cost_volume_fwd(c1, warp, r)[0]


def _costvol_entry(name, r):
    """Entry point and trailing arguments for range r: the range-free (R = 4) entry point for the default range."""
    return (name, ()) if r == 4 else (name + '_r', (r,))


def _cost_volume_fwd(c1, warp, r=4):
    B, h, w, C = c1.shape
    nd = (2 * r + 1) ** 2
    pitch = (nd + 7) // 8 * 8
    a1, a2 = _to_act(c1), _to_act(warp)
    out = torch.zeros(B, h, w, pitch, dtype=torch.bfloat16, device=c1.device)
    op, rng = _costvol_entry('cis_warp_costvol', r)
    _lib.call(op, a1.ptr, a1.pitch, a1.c_off, a2.ptr, a2.pitch, a2.c_off, None, 1.0, B, h, w, C, out.data_ptr(), pitch, 0, *rng, _stream())
    return out[..., :nd].float(), a1, a2


class _CostVolumeFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, c1, warp, r):
        out, a1, a2 = _cost_volume_fwd(c1, warp, r)
        ctx.acts, ctx.r = (a1, a2), r
        ctx.dtypes = (c1.dtype, warp.dtype)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, dout):
        a1, a2 = ctx.acts
        B, h, w, C = a1.N, a1.H, a1.W, a1.C
        d = dout.contiguous().float()
        gs = torch.empty(B, h, w, (2 * ctx.r + 1) ** 2, dtype=torch.float32, device=d.device)
        dc1, dwarp = (torch.empty(B, h, w, C, dtype=torch.float32, device=d.device) for _ in range(2))
        op, rng = _costvol_entry('cis_cost_volume_bwd', ctx.r)
        _lib.call(op, a1.ptr, a1.pitch, a1.c_off, a2.ptr, a2.pitch, a2.c_off, d.data_ptr(), B, h, w, C, gs.data_ptr(),
                  dc1.data_ptr(), dwarp.data_ptr(), *rng, _stream())
        ctx.acts = None
        return tuple(g.to(dt) if n else None for g, dt, n in zip((dc1, dwarp), ctx.dtypes, ctx.needs_input_grad)) + (None,)


def dense_image_warp(image, flow, name=None):
    """models/PWCNet/core_warp.py:153-202 -> image sampled at (y - flow[...,0], x - flow[...,1]), bilinear, edge-clamped.
    Differentiable w.r.t. image (fp64-atomic scatter, rounded to fp32 once) and flow (the clamping rules of core_warp.py)."""
    _check_cuda(image, flow)
    if _needs_grad([image, flow]):
        return _DenseImageWarpFn.apply(image, flow)
    return _dense_image_warp_fwd(image, flow)[0]


def _dense_image_warp_fwd(image, flow):
    B, h, w, C = image.shape
    a = _to_act(image)
    fl = flow.contiguous().float()
    out = torch.zeros(B, h, w, a.pitch, dtype=torch.bfloat16, device=image.device)
    _lib.call('cis_dense_image_warp', a.ptr, a.pitch, a.c_off, fl.data_ptr(), 1.0, B, h, w, C, out.data_ptr(), a.pitch, _stream())
    return out[..., :C].float(), a, fl


class _DenseImageWarpFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, image, flow):
        out, a, fl = _dense_image_warp_fwd(image, flow)
        ctx.act, ctx.flow = a, fl
        ctx.dtypes = (image.dtype, flow.dtype)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, dout):
        a, fl = ctx.act, ctx.flow
        B, h, w, C = a.N, a.H, a.W, a.C
        d = dout.contiguous().float()
        need_img, need_flow = ctx.needs_input_grad[:2]
        dimage = torch.empty(B, h, w, C, dtype=torch.float32, device=d.device) if need_img else None
        scratch = torch.empty(B, h, w, C, dtype=torch.float64, device=d.device) if need_img else None
        dflow = torch.empty(B, h, w, 2, dtype=torch.float32, device=d.device) if need_flow else None
        _lib.call('cis_dense_image_warp_bwd', a.ptr, a.pitch, a.c_off, fl.data_ptr(), 1.0, B, h, w, C, d.data_ptr(), _ptr(dimage),
                  _ptr(scratch), _ptr(dflow), _stream())
        ctx.act = ctx.flow = None
        return tuple(g.to(dt) if g is not None else None for g, dt in zip((dimage, dflow), ctx.dtypes))


# ------------------------------------------------------------------------------------------- convolution_utils.py layer primitives
def elu(x):
    """tf.nn.elu.  Passed as the `activation` of gen_conv / conv it is fused into the conv epilogue (ACT_ELU)."""
    return torch.nn.functional.elu(x)


def leaky_relu(x, alpha=0.2):
    """tf.nn.leaky_relu (alpha = 0.2, TF's default).  Passed as an `activation` it is fused into the conv epilogue (ACT_LEAKY, 0.2)."""
    return torch.nn.functional.leaky_relu(x, alpha)


def identity(x):
    """tf.identity.  Passed as an `activation` the conv has no activation (ACT_NONE)."""
    return x


_FUSED_ACTS = ((elu, _lib.ACT_ELU), (leaky_relu, _lib.ACT_LEAKY), (identity, _lib.ACT_NONE))
LAYER_SUPPORTED = ("square kernels k = 1..7, stride 1 or 2, rate 1..16 with stride 1, padding 'SAME', any Cin >= 1 and Cout >= 1 "
                   "(Cout <= 256 when a gradient is needed)")


def _unsupported(fn, what):
    raise NotImplementedError('%s: %s is not supported; the supported set is %s' % (fn, what, LAYER_SUPPORTED))


def _square(fn, v, what):
    """int or a pair of equal ints (tf.layers accepts both) -> int."""
    if isinstance(v, (list, tuple)):
        if len(v) != 2 or v[0] != v[1]:
            _unsupported(fn, 'non-square %s %r' % (what, tuple(v)))
        v = v[0]
    if isinstance(v, bool) or int(v) != v:
        raise ValueError('%s: %s must be an integer; got %r' % (fn, what, v))
    return int(v)


def _size(fn, size):
    if size is None or len(size) != 2 or any(isinstance(v, bool) or int(v) != v or int(v) < 1 for v in size):
        raise ValueError('%s: size must be two integers >= 1; got %r' % (fn, size))
    return int(size[0]), int(size[1])


def _layer(fn, x, kind, k, cout, stride, rate, padding, activation, name, pre=None, size=None, params=None):
    """Validate one layer call, run it on its _LayerRunner (forward-only plan, or _NetFn when a gradient is needed), apply a non-fused
    activation with torch."""
    if x.dim() != 4:
        raise ValueError('%s: expects an NHWC tensor; got shape %s' % (fn, tuple(x.shape)))
    B, H, W, cin = (int(v) for v in x.shape)
    k, stride, rate = _square(fn, k, 'kernel size'), _square(fn, stride, 'stride'), _square(fn, rate, 'rate')
    if not 1 <= k <= 7:
        _unsupported(fn, 'kernel size %d' % k)
    if stride not in (1, 2):
        _unsupported(fn, 'stride %d' % stride)
    if not 1 <= rate <= 16 or (rate > 1 and stride != 1):
        _unsupported(fn, 'rate %d with stride %d' % (rate, stride))
    if str(padding).upper() != 'SAME':
        _unsupported(fn, 'padding %r' % (padding,))
    if cout < 1 or cin < 1:
        raise ValueError('%s: %d input and %d output channels' % (fn, cin, cout))
    act = next((a for f, a in _FUSED_ACTS if activation is f), None)
    _check_cuda(x)
    sc = str(name).rstrip('/')
    spec = (kind, k, int(cout), stride, rate, _lib.ACT_NONE if act is None else act, pre, size, sc)
    key = (B, H, W, cin) + spec + (str(x.device),)
    make = lambda: _LayerRunner(B, H, W, cin, spec, x.device)
    r = _runner('layer', key, make)
    names, pvals = _param_inputs(r, params)
    for (n, shape, _, _, _), t in zip(r.store.entries, pvals):
        if tuple(t.shape) != shape:
            raise ValueError('%s: parameter %s has shape %s, the call needs %s' % (fn, n, tuple(t.shape), shape))
    if not _needs_grad([x] + pvals):
        y = r(x, params)
    else:
        if cout > 256:
            _unsupported(fn, 'a gradient with Cout %d' % cout)
        lease = _lease('layer', key, make)
        try:
            y = _NetFn.apply(lease, names, 1, x, *pvals)
        except BaseException:
            lease.release()
            raise
    return y if act is not None else activation(y)


def gen_conv(x, cnum, ksize, stride=1, rate=1, name='conv', padding='SAME', activation=elu, training=True, kernel_initializer=None,
             params=None):
    """convolution_utils.py:26-53: conv2d SAME + bias -> inference BN (gamma * x / sqrt(1 + 1e-3) + beta, folded into the weights) ->
    activation.  Parameters <name>/kernel [k,k,Cin,cnum], <name>/bias, <name>/gamma, <name>/beta (name='MaskNet/conv1' reads the
    generator's conv1).  x: fp32 NHWC cuda tensor -> fp32 [B, ceil(H/stride), ceil(W/stride), cnum]; bf16 activations inside, fp32
    gradients w.r.t. x and the four parameters.  elu / leaky_relu / identity are fused; any other callable is applied to the output."""
    return _layer('gen_conv', x, 'gen', ksize, cnum, stride, rate, padding, activation, name, params=params)


def gen_deconv(x, cnum, name='upsample', padding='SAME', training=True, params=None):
    """convolution_utils.py:55-75: nearest-neighbour x2 (align_corners=True), then a 3x3 gen_conv with ELU.  Parameters
    <name>/kernel|bias|gamma|beta (the internal names of MaskNet/conv13_upsample; checkpoint/tf_names.py maps them to TF's
    <name>/<name>_conv/...).  -> fp32 [B, 2H, 2W, cnum]."""
    return _layer('gen_deconv', x, 'gen', 3, cnum, 1, 1, padding, elu, name, pre='nn2x', params=params)


def conv(inputs, name, shape, stride, reuse=None, training=True, activation=leaky_relu, init_w=None, init_b=None, params=None):
    """convolution_utils.py:77-85: tf.nn.conv2d SAME + bias + activation.  shape = [k, k, Cin, Cout]; parameters <name>/weights
    (`shape`) and <name>/biases [Cout]."""
    shape = [int(v) for v in shape]
    if len(shape) != 4:
        raise ValueError('conv: shape must be [k, k, Cin, Cout]; got %r' % (shape,))
    if shape[0] != shape[1]:
        _unsupported('conv', 'non-square kernel %dx%d' % (shape[0], shape[1]))
    if inputs.dim() == 4 and shape[2] != inputs.shape[-1]:
        raise ValueError('conv: shape[2] = %d but the input has %d channels' % (shape[2], inputs.shape[-1]))
    return _layer('conv', inputs, 'conv', shape[0], shape[3], stride, 1, 'SAME', activation, name, params=params)


def deconv(inputs, size, name, shape, reuse=None, training=True, activation=leaky_relu, params=None):
    """convolution_utils.py:87-90: legacy bilinear resize (tf.image.resize_images, align_corners=False) to `size` = [h, w], then conv
    with stride 1.  Parameters <name>/weights (`shape`) and <name>/biases."""
    shape = [int(v) for v in shape]
    if len(shape) != 4:
        raise ValueError('deconv: shape must be [k, k, Cin, Cout]; got %r' % (shape,))
    if shape[0] != shape[1]:
        _unsupported('deconv', 'non-square kernel %dx%d' % (shape[0], shape[1]))
    if inputs.dim() == 4 and shape[2] != inputs.shape[-1]:
        raise ValueError('deconv: shape[2] = %d but the input has %d channels' % (shape[2], inputs.shape[-1]))
    return _layer('deconv', inputs, 'conv', shape[0], shape[3], 1, 1, 'SAME', activation, name, pre='bilinear',
                  size=_size('deconv', size), params=params)


def resize_bilinear(x, size, align_corners=False, name=None):
    """tf.image.resize_bilinear (TF 1.13, no half-pixel centres) on fp32 NHWC: step (in-1)/(out-1) with align_corners and out > 1, else
    in/out; lo = floor(d * step), hi = min(lo + 1, in - 1).  Any sizes, up or down.  Differentiable w.r.t. x (a deterministic gather)."""
    return _resize('resize_bilinear', x, size, _lib.RESIZE_BILINEAR, align_corners)


def resize_nearest_neighbor(x, size, align_corners=False, name=None):
    """tf.image.resize_nearest_neighbor (TF 1.13) on fp32 NHWC: source index roundf(d * step) with align_corners, floor(d * step)
    without, clamped to in - 1.  Any sizes.  Differentiable w.r.t. x (a deterministic gather)."""
    return _resize('resize_nearest_neighbor', x, size, _lib.RESIZE_NEAREST, align_corners)


def resize(x, scale=2, to_shape=None, align_corners=True, dynamic=False, func=resize_bilinear, name='resize'):
    """convolution_utils.py:4-24: func(x, [int(H * scale), int(W * scale)] or to_shape[:2], align_corners=align_corners); any callable
    with that signature runs as it is."""
    size = [int(x.shape[1] * scale), int(x.shape[2] * scale)] if to_shape is None else [to_shape[0], to_shape[1]]
    return func(x, size, align_corners=align_corners)


def _resize(fn, x, size, method, align_corners):
    if x.dim() != 4:
        raise ValueError('%s: expects an NHWC tensor; got shape %s' % (fn, tuple(x.shape)))
    oh, ow = _size(fn, size)
    _check_cuda(x)
    ac = 1 if align_corners else 0
    if _needs_grad([x]):
        return _ResizeFn.apply(x, oh, ow, method, ac)
    return _resize_fwd(x, oh, ow, method, ac)


def _resize_fwd(x, oh, ow, method, ac):
    N, H, W, C = x.shape
    xs = x.contiguous().float()
    out = torch.empty(N, oh, ow, C, dtype=torch.float32, device=x.device)
    _lib.call('cis_resize_f32', xs.data_ptr(), N, H, W, C, out.data_ptr(), oh, ow, method, ac, _stream())
    return out


class _ResizeFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, oh, ow, method, ac):
        ctx.meta = (tuple(x.shape), x.dtype, oh, ow, method, ac)
        return _resize_fwd(x, oh, ow, method, ac)

    @staticmethod
    @once_differentiable
    def backward(ctx, dout):
        (N, H, W, C), dt, oh, ow, method, ac = ctx.meta
        d = dout.contiguous().float()
        dx = torch.empty(N, H, W, C, dtype=torch.float32, device=d.device)
        _lib.call('cis_resize_f32_bwd', d.data_ptr(), N, oh, ow, C, H, W, dx.data_ptr(), method, ac, _stream())
        return dx.to(dt), None, None, None, None


# ---------------------------------------------------------------------------------------------------------- flow_utils.py
def preprocess_flow_batch(flow):
    """flow_utils.py:5-12: (flow - mean) / sqrt(variance) per sample and channel over H x W (population variance, no epsilon) for fp32
    [B,H,W,2] flows -- the standardisation in front of generator_net.  Differentiable w.r.t. flow: dx = (g - mean(g) - y mean(g y)) / sigma
    with fixed-order reductions (bit-identical run to run)."""
    if flow.dim() != 4 or flow.shape[-1] != 2:
        raise ValueError('preprocess_flow_batch: expects a [B,H,W,2] flow; got shape %s' % (tuple(flow.shape),))
    _check_cuda(flow)
    if _needs_grad([flow]):
        return _FlowStdFn.apply(flow)
    return _flow_std_fwd(flow)[0]


def _flow_std_fwd(flow):
    B, H, W, _ = flow.shape
    f = flow.contiguous().float()
    stats = torch.zeros(B, 4, dtype=torch.float64, device=f.device)
    out = torch.empty_like(f)
    _lib.call('cis_flow_stats', f.data_ptr(), B, H * W, stats.data_ptr(), _stream())
    _lib.call('cis_flow_standardize', f.data_ptr(), stats.data_ptr(), B, H * W, out.data_ptr(), _stream())
    return out, stats


class _FlowStdFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, flow):
        out, stats = _flow_std_fwd(flow)
        ctx.y, ctx.stats, ctx.dtype = out, stats, flow.dtype
        return out.clone()

    @staticmethod
    @once_differentiable
    def backward(ctx, dout):
        y, stats = ctx.y, ctx.stats
        B, H, W, _ = y.shape
        d = dout.contiguous().float()
        scratch = torch.empty(B * 256, dtype=torch.float64, device=d.device)
        dx = torch.empty_like(y)
        _lib.call('cis_flow_standardize_bwd', y.data_ptr(), d.data_ptr(), stats.data_ptr(), B, H * W, scratch.data_ptr(), dx.data_ptr(),
                  _stream())
        ctx.y = ctx.stats = None
        return dx.to(ctx.dtype)
