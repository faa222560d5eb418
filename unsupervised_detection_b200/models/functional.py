"""Function-level surface of the reference on top of the launch-list engine (SURVEY 8b: `generator_net`, `recover_net`,
`charbonnier_loss`, `train_op`, `cost_volume`, `dense_image_warp`, `ModelPWCNet.predict_from_img_pairs` keep their names and NHWC
argument order; TF-only arguments -- scope / reuse / name / training -- are accepted, `scope` selects the parameter-name prefix).

The reference functions create TF graph nodes; here each call runs the corresponding sub-graph of libcis_b200 kernels on `cuda`
tensors and returns a device tensor.  Static launch plans are cached per input shape; parameters come from the `params` argument or
from the registry filled by `set_parameters()` (dict name -> tensor, names as in oracle/params.py / a loaded checkpoint).
PyTorch is used for memory and the small amount of buffer plumbing only; there is no CPU fallback: without the CUDA library (or on CPU
tensors) the calls raise.

STATUS: the sub-graphs reuse the builders that the step graph is made of; the GPU tests of these wrappers
(tests/test_functional_api_gpu.py) are gated behind CIS_TEST_EXPERIMENTAL=1; tests/test_functional_api_cpu.py checks the plumbing
with a recording stub.
"""
import torch

from .. import _lib
from ..engine import Act, Builder, ParamStore, Plan
from .nets import GeneratorNet, RecoverNet

_PARAMS = {}
_RUNNERS = {}


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
    """One cached static plan: parameter store + packed operands + input/output buffers for a fixed shape."""

    def __init__(self, device):
        self.device = device
        self.store = ParamStore(device)
        self.bld = Builder(device)
        self.pack = Plan('pack')
        self.dirty = True
        self._loaded = None

    def finish(self, layers):
        for L in layers:
            L.plan_pack(self.pack)

    def load(self, params):
        src = params if params is not None else _PARAMS
        if self.dirty or self._loaded is not src:
            self.store.load(src)
            self.pack.run()
            self.dirty, self._loaded = False, src


class _GeneratorRunner(_NetRunner):
    def __init__(self, B, H, W, device, scope):
        _NetRunner.__init__(self, device)
        self.net = GeneratorNet(self.store, scope)
        self.store.finalize(False)
        f32 = self.bld.f32
        self.image, self.flow, self.mask = f32(B, H, W, 3), f32(B, H, W, 2), f32(B, H, W, 1)
        # generator_net receives the ALREADY normalised flow (adversarial_learner.py:100-105); cis_pack_generator_input normalises with
        # the statistics it is given, so feed it mean 0 / variance 1: {sum, sum, sum of squares, sum of squares} = {0, 0, hw, hw}
        self.stats = torch.tensor([[0.0, 0.0, float(H * W), float(H * W)]] * B, dtype=torch.float64, device=device)
        self.gen_in = self.bld.new_act(B, H, W, 5, name='gen_in')
        self.bld.fwd.add('cis_pack_generator_input', self.image.data_ptr(), self.flow.data_ptr(), self.stats.data_ptr(), B, H * W, self.gen_in.ptr)
        self.net.build(self.bld, self.gen_in, self.mask)
        self.finish(self.net.all_layers())

    def __call__(self, images, flows, params):
        self.load(params)
        self.image.copy_(images)
        self.flow.copy_(flows)
        self.bld.fwd.run()
        return self.mask.clone()


class _RecoverRunner(_NetRunner):
    def __init__(self, B, H, W, device, scope, f):
        _NetRunner.__init__(self, device)
        self.net = RecoverNet(self.store, scope, f)
        self.store.finalize(False)
        f32 = self.bld.f32
        self.B, self.H, self.W = B, H, W
        self.h1, self.w1 = -(-H // 2), -(-W // 2)
        self.image, self.aug = f32(B, H, W, 3), f32(B, H, W, 4)
        self.flow1, self.pred = f32(B, self.h1, self.w1, 2), f32(B, H, W, 2)
        self.img8 = self.bld.new_act(B, H, W, 3, name='img8')
        self.flow_in = self.bld.new_act(B, H, W, 4, name='rec_in')
        P = self.bld.fwd
        P.add('cis_pack_f32_to_bf16', self.image.data_ptr(), B * H * W, 3, 0.0, self.img8.ptr, 8, 0)
        P.add('cis_pack_f32_to_bf16', self.aug.data_ptr(), B * H * W, 4, 0.0, self.flow_in.ptr, 8, 0)
        self.net.build(self.bld, self.img8, self.flow_in, self.flow1, ncalls=1)
        P.join()
        P.add('cis_resize_bilinear_f32', self.flow1.data_ptr(), B, self.h1, self.w1, 2, self.pred.data_ptr(), H, W, 1.0)   # nets.py:108
        self.finish(self.net.all_layers())

    def __call__(self, img1, flow_masked, mask, params):
        self.load(params)
        self.image.copy_(img1)
        # input augmentation of nets.py:50-53: [flow_masked, ones, 1 - mask]
        self.aug[..., 0:2].copy_(flow_masked)
        self.aug[..., 2:3].fill_(1.0)
        self.aug[..., 3:4].copy_(1.0 - mask)
        self.bld.fwd.run()
        return self.pred.clone()


class _PWCRunner(_NetRunner):
    def __init__(self, B, H, W, device, name):
        from .PWCNet.model_pwcnet import ModelPWCNet
        _NetRunner.__init__(self, device)
        self.net = ModelPWCNet(self.store, name)
        self.store.finalize(False)
        f32 = self.bld.f32
        self.img1, self.img2, self.flow = f32(B, H, W, 3), f32(B, H, W, 3), f32(B, H, W, 2)
        i1, i2 = self.bld.new_act(B, H, W, 3, name='img1_8'), self.bld.new_act(B, H, W, 3, name='img2_8')
        P = self.bld.fwd
        P.add('cis_pack_f32_to_bf16', self.img1.data_ptr(), B * H * W, 3, 0.5, i1.ptr, 8, 0)      # adapt_x: images arrive in [-0.5, 0.5]
        P.add('cis_pack_f32_to_bf16', self.img2.data_ptr(), B * H * W, 3, 0.5, i2.ptr, 8, 0)
        self.net.build(self.bld, i1, i2, self.flow)
        self.finish(self.net.all_layers())

    def __call__(self, img1, img2, params):
        self.load(params)
        self.img1.copy_(img1)
        self.img2.copy_(img2)
        self.bld.fwd.run()
        return self.flow.clone()


def _runner(kind, key, make):
    k = (kind,) + key
    r = _RUNNERS.get(k)
    if r is None:
        _lib.load()
        r = _RUNNERS[k] = make()
    return r


# ------------------------------------------------------------------------------------------------------------------ networks
def generator_net(images, flows, scope='MaskNet', reuse=None, training=True, params=None):
    """models/nets.py:4-42 -> generated mask [B,H,W,1] in (0,1).  images [B,H,W,3] in [-0.5,0.5], flows [B,H,W,2] normalised."""
    _check_cuda(images, flows)
    B, H, W, _ = images.shape
    sc = _scope_name(scope, 'MaskNet')
    r = _runner('gen', (B, H, W, str(images.device), sc), lambda: _GeneratorRunner(B, H, W, images.device, sc))
    return r(images, flows, params)


def recover_net(img1, flow_masked, mask, scope='FlownetS', reuse=None, f=0.25, training=True, params=None):
    """models/nets.py:45-110 -> recovered flow [B,H,W,2] at the input resolution."""
    _check_cuda(img1, flow_masked, mask)
    B, H, W, _ = img1.shape
    sc = _scope_name(scope, 'FlownetS')
    r = _runner('rec', (B, H, W, str(img1.device), sc, f), lambda: _RecoverRunner(B, H, W, img1.device, sc, f))
    return r(img1, flow_masked, mask, params)


def predict_from_img_pairs(img1, img2, name='pwcnet', params=None):
    """ModelPWCNet.predict_from_img_pairs (model_pwcnet.py:39-76): forward flow img1 -> img2, [B,H,W,2] in pixels of the input size
    (H, W multiples of 64, 384x640 in the reference's pipeline)."""
    _check_cuda(img1, img2)
    B, H, W, _ = img1.shape
    if H % 64 or W % 64:
        raise ValueError('PWC-Net needs input sizes that are multiples of 64 (6 pyramid levels); got %dx%d' % (H, W))
    r = _runner('pwc', (B, H, W, str(img1.device), name), lambda: _PWCRunner(B, H, W, img1.device, name))
    return r(img1, img2, params)


# -------------------------------------------------------------------------------------------------------------------- losses
def charbonnier_loss(gt_flows, pred_flows, masks, cbn=0.5):
    """models/utils/loss_utils.py:34-51 -> [B]: sum over H, W, C of ((gt - pred)^2 + 0.001^2)^cbn * mask."""
    _check_cuda(gt_flows, pred_flows, masks)
    B, H, W, C = gt_flows.shape
    mc = masks.shape[-1]
    if tuple(masks.shape[:3]) != (B, H, W) or mc not in (1, C) or tuple(pred_flows.shape) != (B, H, W, C):
        raise ValueError('charbonnier_loss: shapes %s / %s / %s' % (tuple(gt_flows.shape), tuple(pred_flows.shape), tuple(masks.shape)))
    g, p, m = (t.contiguous().float() for t in (gt_flows, pred_flows, masks))
    sums = torch.zeros(B, dtype=torch.float64, device=g.device)
    _lib.call('cis_charbonnier_sum', g.data_ptr(), p.data_ptr(), m.data_ptr(), B, H * W, C, mc, float(cbn), sums.data_ptr(), _stream())
    return sums.float()


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
    """models/PWCNet/core_costvol.py:20-40 -> [B,h,w,(2r+1)^2]: leaky_relu(mean_c c1 * shifted warp, 0.1), zero padded, dy outer.
    The kernel is built for the reference's search_range = 4 (81 displacements); features and result are bf16-rounded like in the
    pipeline."""
    _check_cuda(c1, warp)
    if search_range != 4:
        raise NotImplementedError('cost_volume: the fused kernel implements search_range=4 (model_pwcnet.py options)')
    B, h, w, C = c1.shape
    a1, a2 = _to_act(c1), _to_act(warp)
    out = torch.zeros(B, h, w, 88, dtype=torch.bfloat16, device=c1.device)
    _lib.call('cis_warp_costvol', a1.ptr, a1.pitch, a1.c_off, a2.ptr, a2.pitch, a2.c_off, None, 1.0, B, h, w, C, out.data_ptr(), 88, 0, _stream())
    return out[..., :81].float()


def dense_image_warp(image, flow, name=None):
    """models/PWCNet/core_warp.py:153-202 -> image sampled at (y - flow[...,0], x - flow[...,1]), bilinear, edge-clamped."""
    _check_cuda(image, flow)
    B, h, w, C = image.shape
    a = _to_act(image)
    fl = flow.contiguous().float()
    out = torch.zeros(B, h, w, a.pitch, dtype=torch.bfloat16, device=image.device)
    _lib.call('cis_dense_image_warp', a.ptr, a.pitch, a.c_off, fl.data_ptr(), 1.0, B, h, w, C, out.data_ptr(), a.pitch, _stream())
    return out[..., :C].float()
