"""Every non-convolution launch of a launch plan (resampling, concatenation, activation derivatives, bias-gradient partials, residual
gradients, warp + cost volume, input packing), checked on its own against a float64 reference of the same operation.  The counterpart of
tests/conv_launch_ref.py; `Walker(rec, glue=Glue())` replays a plan once with both checkers.

Operands come from the launch arguments, not from the builders
    Each op's argument tuple is decoded against the C ABI (include/cis_b200.h; ARGS below names every argument, in order).  Pointers are
    resolved to the live CUDA storage that contains them (an interval search) and viewed with the pitches, channel offsets, row counts,
    CisSrc arrays and want / accumulate arrays the launch passes.  A wrong pitch, offset, row count or accumulate flag from a builder is
    caught like a wrong kernel.  Before the launch the checker reads the operands and snapshots every destination storage; after it, it
    synchronises and compares.  Acts found on the heap give the channel maps, for the padding-channel check.

Per-element bound, no normalisation by the tensor maximum (the form of conv_launch_ref):

    |got - ref| <= e_out |ref| + gamma S + delta,     e_out = 2^-8 for bf16 stores, 0 for fp32 ones; u = 2^-24 below.

  Bit-exact (torch.equal against the restated gather or rounding): cis_zero, cis_pack_f32_to_bf16 (the fp32 add of `offset`, then round to
    nearest), cis_cast_bf16_to_f32, cis_parity_split_bf16, cis_upsample_nn2x (source index min(roundf(d * fp32((n-1)/(2n-1))), n-1); no
    product lands on a .5 tie at these sizes, which is asserted), same-resolution cis_resize_concat_bf16, cis_add_slice (sequential fp32
    sum of the accumulate term and the reps sources, then bf16), and the gradient cis_dact_mul / cis_dact_colsum write: bf16(g * d(u)),
    u = y - res formed in fp32 from the bf16 values read, d = 1 for u > 0, else u + 1 (ELU) or alpha (leaky), in fp32.  The branch is exact:
    the fp32 difference of two bf16 values keeps its sign.
  Legacy bilinear (cis_resize_bilinear_f32, the x2 and generic cis_resize_concat_bf16, cis_resize_bilinear_bf16): the source position
    d * fp32(in / out) in fp32, as the kernels take it (tests/resize_ref.py), the interpolation in fp64.  Each fp32 lerp t = a + (b - a) f
    adds at most u (|a| + |b|) per rounding, three roundings, and the second lerp takes two such values with weights <= 1; the `scale`
    multiply adds u |result|.  So gamma = 2^-21 on S = the sum of the four |corner| values (times |scale|), FMA contraction included.
  Transposes (cis_resize_concat_bf16_bwd, cis_resize_bilinear_bf16_bwd, cis_upsample_nn2x_bwd, cis_resize_f32_bwd_to_bf16_scaled): fp64
    transpose of the forward restatement, replicas of batch-broadcast sources folded, plus the snapshot where the launch accumulates.
    gamma = (terms + 1) 2^-23 per element, terms = the nonzero weights of that element times the replicas; S = the same transpose of |dd|
    plus |snapshot|.  The fp32 weight products wy * wx and 1 - f add <= 3u per term, inside the +1 and the factor two.
  Column sums (cis_colsum, the partials of cis_dact_colsum): the sum over the launch's nblk partial rows against the fp64 column sum of
    the (rounded) gradient.  A block's partial goes through ceil(npix / (nblk P)) lane additions and P lane-reduction additions
    (P = 256 / chunks pixel lanes): gamma = (that + P) 2^-23, S = sum |g|.
  cis_flow_stats: the four fp64 sums against fp64 sums of the flow read, after the zeroed snapshot; gamma = (hw + 64) 2^-53.
  cis_pack_generator_input: channels 0-2 = bf16(image) exactly, 5-7 exactly 0, 3-4 against oracle.losses.preprocess_flow_batch of the
    flow read (fp64); the kernel's fp32 (f - m) * r adds <= 3u (|f| + |m|) r: gamma = 2^-21 on S = (|f| + |m|) r.
  cis_warp_costvol: q = grid - fs * flow in fp64 from the fp32 flow; bilinear with the kernel's clamps (floor clamped to [0, size-2], alpha
    to [0, 1]), zero outside the image, the mean over the real C, leaky 0.1, bf16.  The fp32 position may be rounded or contracted:
    eps_q = 2^-23 (|q| + |fs flow|) per axis.  Bilinear is continuous in q, so the warped value moves by <= eps_q 2 M, M = max |c2| over
    the 4 x 4 neighbourhood of the cell; with the lerps' 2^-21 sum |corners| this is Werr.  The correlation sums Cp products in fp32:
    bound_pre = (Cp + 6) 2^-23 S_pre + corr(|c1|, Werr) / C (the 1 / C multiply inside the +6).  Where |pre_ref| <= bound_pre either
    slope of the leaky is accepted.  The bound is per (pixel, displacement), so it does not depend on the search range R.  The window is
    the (2R+1)^2 channels at `oo`, dy outer, padded to a multiple of 8; the padding channels must be +0 bit for bit (at R = 1 a compact
    16-channel conv reads all 16), and outside the window the destination is bit-identical.  At R = 4 too: channels 81-87 lie inside the
    88-channel window, where they are held to +0 instead of to their bits before the launch.
  cis_warp_costvol_r, cis_warp_costvol_bwd_r: the same references with R = the trailing argument r (1 .. 4): (2r+1)^2 = 9 / 25 / 49
    channels in windows of 16 / 32 / 56 for r = 1 / 2 / 3.
  cis_warp_costvol_bwd: the same composite transposed in fp64 (dc1 = sum_d g' warp[p+d], dwarp = sum_d g'[q-d] c1[q-d], dc2 = the
    bilinear scatter of dwarp, d(flow) = -fs sum_c dwarp (d warp / dq), zero where q - floor leaves [0, 1]), acc bits honoured.  The gate
    is recomputed in fp32, so the (pixel, displacement) pairs with |pre_ref| <= bound_pre may be gated either way: their contribution at
    slope difference 0.9 joins delta.  gamma = (ND + 6) 2^-23 (the ND-term sums, fp32 scratch), times the bilinear weights for dc2.  The
    flow gradient jumps where q crosses an integer (a clamp edge is one): positions within eps_q of one take 4 M |dwarp| fs per channel
    into delta, and their scatter is spread over the 4 x 4 neighbourhood.

The PWC-Net training step (FlowTrainGraph; the kernels in csrc/misc_kernels.cu, built without --use_fast_math: sqrtf and division are
correctly rounded, powf within CUDA's documented 4 ulp, rsqrtf and expf within 2 ulp).  U = 2^-24 is fp32's unit roundoff.
  cis_flow_multiscale_loss: the [B, 5] sums against fp64 sums of rho(flow_l - g_l), g_l the legacy-bilinear sample of gt (fp32 source
    positions, as lerp_axis forms them) times fp32(s_c) 2^-l.  The kernel's fp32 difference is within e_c = 2^-21 S_c |s_c 2^-l| + 2^-23
    (|flow_c| + |g_c|) per channel (the lerps and the scale product as for cis_resize_bilinear_f32, then the subtraction).  ||.|| is
    1-Lipschitz: rho moves by <= e_0 + e_1; robust rho by <= q max(x - E, eps)^(q-1) E, x = |d_0| + |d_1| + eps, E = e_0 + e_1 (the
    local derivative at the interval's low end).  The sums are fp64: + (hw + 128) 2^-53 sum rho.  scratch and out are destinations.
  cis_flow_multiscale_loss_bwd: the five bf16 level gradients weight[i] d rho / d flow (+ the snapshot where accumulate[i]).  ||.||:
    d / ||d|| moves by <= 2 ||e|| / ||d||, + 2^-21 for the fp32 squares, sum, sqrtf, division and weight product; where ||d|| <= 4 E any
    vector of norm <= weight is accepted.  Robust: k = q powf(x, q - 1) with x within E + 2^-23 x, so k within q (1 - q) x_lo^(q-2) (that)
    + k (4 2^-23 + 2^-24 + |ln x| 2^-24) (powf, the product, the fp32 exponent q - 1); a component with |d_c| <= e_c may take either sign
    or 0.  Destinations are exactly [c_off, c_off + 2) of each level; the padding channels of the level-gradient buffers must be +0 after
    the launch (up_flow's data gradient and the predict-flow convs read them).
  cis_adam_l2: fp64 TF-Adam from snapshots of param, m, v, grad, lr and step, decay inside the decoded segments only.  Per element, from
    the fp32 operation count: e_g = U (2 |decay w| + |g|), e_m = 2U (b1 |m| + (1 - b1) |g|) + (1 - b1) e_g, e_v = 3U (b2 v + (1 - b2) g^2)
    + 2 (1 - b2) |g| e_g; lr_t relative 2^-23 / (1 - b2^t) + 2^-22 / (1 - b1^t) + 4U (powf's 4 ulp on b^t in [0.5, 1), 1 - b^t exact by
    Sterbenz, sqrtf, two products); sqrt(v') + eps within min(e_v / (2 sqrt v'), sqrt e_v) + 2U (sqrt v' + eps); the update
    lr_t m' / (sqrt v' + eps) relative (that + 3U) plus lr_t e_m / (sqrt v' + eps); the parameter + U |w'|.  step_state must advance by
    exactly 1 and grad stay bit-identical.
  cis_flow_aug_params: flow_aug_ref's draw from the decoded ranges, seed and sample_offset at the step read from step_state before the
    launch.  The accepted attempt (26), the noise key (25, as uint32) and the zero tail are bit-identical; columns 0-24 within one fp32 ulp
    of fp32(the fp64 value) (the ratio is in ulps).
  cis_flow_augment: flow_aug_ref.augment's fp64 per-pixel pass for both frames and the flow, within flow_aug_ref.tolerances (the bounds
    tests/test_flow_aug_gpu.py uses too: fp32 sample positions through the Lipschitz bound of the sampled field and the photometric chain;
    the flow through T2^-1's row norm).
  cis_unsup_flow_loss: the occlusion test runs in fp32 on the partner flow h sampled at q (lerps and fp32 alphas: 2^-20 sum |corners|
    = eh per channel), so lhs = |f + h|^2 and rhs = 0.01f (|f|^2 + |h|^2) + 0.5f are within e_lhs = sum_c 2 |s_c| (eh_c + 2^-23 |s_c|)
    + eh_c^2 + 3 2^-23 lhs and e_rhs = 0.01 sum_c (2 |h_c| eh_c + eh_c^2) + |0.01f - 0.01| (|f|^2 + |h|^2) + 6 2^-23 rhs; the mask must be
    the fp64 one except where |lhs - rhs| <= 2 (e_lhs + e_rhs).  The frame-border test is exact: q = p - F is formed in double from the
    fp32 flow by the kernel and the reference alike.  Where the mask is ambiguous the references use the launch's own bit.  warped: the
    fp64 sample of the gray levels, within 2^-20 sum |corners| (fp32 gray levels and alphas, the lerps).  The census is recomputed from
    the launch's own warped (checked above) and the fp64 gray levels of S; c within e_c (_census_bound: the fp32 rounding of the gray
    levels and differences through t's slope, t within 8U |t|, e = t_S - t_T through phi's largest slope on the interval, phi within 8U
    phi, the 48-term fp32 sum).  psi = powf(c + 0.01f, 0.4f) within 0.4 c_lo^-0.6 Dc + psi (|ln(c + 0.01)| |0.4f - 0.4| + 4 2^-23), Dc =
    e_c + 2^-23 (c + 0.01) + |0.01f - 0.01|, c_lo = max(c - Dc, 0) + 0.01; coef = M 0.4f powf(c + 0.01f, -0.6f) likewise (slope 0.24
    c_lo^-1.6).  Smoothness: w within rel_w = 5 (e/3) 8U + 3 2^-23 (fp32 differences, the 1/3f and -10 products, expf), l in double as
    the kernel forms it; where |l_c| is within 2^-50 (|a| + 2|b| + |c|) of the ROUNDING threshold w |l_c| joins delta.  Sums fp64:
    + (hw + 128) 2^-53 sum M psi and (2 hw + 128) 2^-53 sum w s.
  cis_unsup_flow_loss_bwd: checked on its own from the forward's warped and coef buffers.  Reference: unsup_bwd_gather, the explicit
    fp64 gather (test_flow_train_launches_cpu.py proves it equals autograd of unsup_flow_loss_ref).  Per window term (k(r+d) + k(r)) h,
    h = -0.2 e / (0.1 + e^2)^2 0.81 iu^3: the fp32 e within e_e (as in the forward) through |dh/de| <= 0.2 (0.1 + 3x) / (0.1 + x)^3
    0.81 iu^3 at x = max(|e| - e_e, 0)^2 (it falls with x), and 33 U |h| for the term's own fp32 operations; the 48-term sum 48 2^-23
    sum |terms| (S: the same gather over |terms|); the chain factor (bot - top etc.) within 2^-20 sum |corners|.  The sample point q is
    exact in double on both sides, so floor, clamps and pass flags agree and no jump enters delta.  Smoothness: w rel_w per stencil term,
    6 2^-23 sum |c w| for the fp32 sum, |c w| where the centre's sign is ambiguous.  Then 2^-23 |dflow| for the final additions.

Stray writes: every destination storage is snapshotted whole; after the launch every byte outside the windows the launch owns (rows x
channel window of each destination) must be unchanged, and the padding channels inside the windows (padding in every Act that views the
buffer) must be exactly 0.

Negative controls (a ratio > 1 means the bound rejected the corruption); they act on the reference or on a copy of the result only:
  resize.row_off_by_one, rc_bwd.fold_dropped, rc_bwd.overwrite, dact.d_at_y, colsum.block_dropped, add_slice.acc_dropped,
  warp_costvol.fs_x1.25, warp_costvol_r1.dx_outer (the r = 1 cost volume with its displacements listed dx outer), costvol_bwd.gate_one,
  and tile.<entry point>: one 16 x 8 tile of one channel of a bf16 result scaled by 1 + 2^-5.
  The training step's: ms_loss.axes_swapped (s0 and s1 exchanged; only made where they differ), ms_loss.level_scale (targets at
  2^-(l-1)), ms_loss_bwd.weights_reversed, unsup.mask_ones, unsup_bwd.smooth_dropped, aug_params.step_frozen (rows drawn at step 0, made
  from step 1 on), augment.flow_unmapped (the flow resampled at T1 but not passed through T2^-1), adam.decay_everywhere and
  adam.t_off_by_one (made from t = 2 on).  pack.unswapped lives in tests/test_flow_train_launches_gpu.py.
"""
import bisect
import collections
import gc

import torch
import torch.nn.functional as F

from oracle import losses as OL
from unsupervised_detection_b200 import engine as E
from unsupervised_detection_b200 import _lib
from unsupervised_detection_b200._lib import ACT_ELU

U23 = 2.0 ** -23
E_BF16 = 2.0 ** -8
FLOOR = 2.0 ** -100
G_LERP = 2.0 ** -21

# the C ABI arguments of every entry point this module checks, in order (the trailing stream is not listed)
ARGS = {
    'cis_zero': 'ptr nbytes',
    'cis_pack_f32_to_bf16': 'src npix C offset dst dp dc',
    'cis_cast_bf16_to_f32': 'src npix pitch coff C dst',
    'cis_parity_split_bf16': 'src sp sc N H W C dst dp',
    'cis_upsample_nn2x': 'src N H W pitch dst',
    'cis_upsample_nn2x_bwd': 'dd N H W pitch ds acc',
    'cis_resize_bilinear_f32': 'src N H W C dst OH OW scale',
    'cis_resize_bilinear_bf16': 'src sp sc N H W dst dp dc OH OW chunks',
    'cis_resize_bilinear_bf16_bwd': 'dd dp dc N OH OW ds sp sc H W chunks acc',
    'cis_resize_concat_bf16': 'srcs nsrc N H W dst dp dc OH OW',
    'cis_resize_concat_bf16_bwd': 'dd dp dc N OH OW grads want acc nsrc H W',
    'cis_resize_f32_bwd_to_bf16_scaled': 'dd N OH OW C H W ds sp scale',
    'cis_dact_mul': 'g gp gc y yp yc res rp rc npix chunks act alpha',
    'cis_dact_colsum': 'g gp gc y yp yc res rp rc npix nch act alpha part nblk',
    'cis_colsum': 'g gp gc npix nch part nblk',
    'cis_add_slice': 'dst dp dc src sp sc npix chunks reps acc',
    'cis_flow_stats': 'flow B hw stats',
    'cis_pack_generator_input': 'image flow stats B hw dst',
    'cis_warp_costvol': 'c1 c1p c1o c2 c2p c2o flow fs B h w C out op oo',
    'cis_warp_costvol_bwd': 'c1 c1p c1o c2 c2p c2o flow fs B h w C dcorr dcp dco dc1 dc1p dc1o dc2 dc2p dc2o dflow dfp dfo acc gs ws ds',
    'cis_warp_costvol_r': 'c1 c1p c1o c2 c2p c2o flow fs B h w C out op oo r',
    'cis_warp_costvol_bwd_r': 'c1 c1p c1o c2 c2p c2o flow fs B h w C dcorr dcp dco dc1 dc1p dc1o dc2 dc2p dc2o dflow dfp dfo acc gs ws ds '
                              'r',
    # the PWC-Net training step (FlowTrainGraph)
    'cis_flow_multiscale_loss': 'pyr gt B H W GH GW s0 s1 robust eps q scratch out',
    'cis_flow_multiscale_loss_bwd': 'pyr gt B H W GH GW s0 s1 robust eps q',
    'cis_unsup_flow_loss': 'flow img1 img2 B H W warped mask coef scratch out',
    'cis_unsup_flow_loss_bwd': 'flow img1 img2 B H W warped coef w_photo w_smooth dflow',
    'cis_flow_aug_params': 'ranges B H W sample_offset step seed params',
    'cis_flow_augment': 'img1 img2 gt params B H W img1_out img2_out gt_out',
    'cis_adam_l2': 'param m v grad n seg nseg decay lr beta1 beta2 eps step_state',
}

# entry points of the step pinned per launch by other tests (the ownership test of tests/test_glue_launches_cpu.py)
PINNED_ELSEWHERE = {
    'cis_cis_loss_fwd': 'tests/test_loss_head_gpu.py', 'cis_cis_loss_reduce': 'tests/test_loss_head_gpu.py',
    'cis_cis_loss_bwd': 'tests/test_loss_head_gpu.py', 'cis_mask_apply': 'tests/test_loss_head_gpu.py',
    'cis_mask_bwd': 'tests/test_loss_head_gpu.py', 'cis_resize_f32_bwd_to_bf16': 'tests/test_loss_head_gpu.py',
    'cis_grad_avg_abs': 'tests/test_loss_head_gpu.py', 'cis_clip_adam': 'tests/test_loss_head_gpu.py',
    'cis_box_masks': 'tests/test_recover_pretrain_gpu.py',
}
CONV_WALKER = {'cis_conv_igemm', 'cis_conv_wgrad', 'cis_param_multi'}
STRUCTURAL = {'join', 'take_stage'}


def decode(op):
    """The argument dict of a glue op (names of ARGS)."""
    names = ARGS[op[2]].split()
    assert len(names) == len(op[1]), (op[2], len(op[1]))
    return dict(zip(names, op[1]))


# ------------------------------------------------------------------------------------------------------------ device memory
class Mem(object):
    """Live CUDA storages by address (interval search), and the Acts that view them."""

    def __init__(self):
        self.refresh()

    def refresh(self):
        spans = {}
        acts = collections.defaultdict(list)
        for o in gc.get_objects():
            t = type(o)
            if t in (torch.Tensor, torch.nn.Parameter):
                if o.is_cuda:
                    st = o.untyped_storage()
                    if st.nbytes():
                        spans[st.data_ptr()] = st
            elif t is E.Act:
                if o.buf.is_cuda:
                    acts[(o.ptr, o.pitch)].append(o)
        self.starts = sorted(spans)
        self.st = [spans[p] for p in self.starts]
        self.acts = acts

    def _find(self, p):
        i = bisect.bisect_right(self.starts, p) - 1
        if i < 0 or p >= self.starts[i] + self.st[i].nbytes():
            return None
        return i

    def storage(self, p):
        """(uint8 tensor over the whole storage holding address p, byte offset of p)."""
        i = self._find(p)
        if i is None:
            self.refresh()
            i = self._find(p)
            if i is None:
                raise ValueError('pointer 0x%x is in no live CUDA storage' % p)
        st = self.st[i]
        t = torch.empty(0, dtype=torch.uint8, device='cuda').set_(st, 0, (st.nbytes(),))
        return t, p - self.starts[i]

    def view(self, p, dtype, shape):
        t, off = self.storage(p)
        n = dtype.itemsize
        for s in shape:
            n *= s
        assert off + n <= t.numel(), ('view past the end of its storage', hex(p), dtype, shape)
        return t[off:off + n].view(dtype).view(shape)

    def pads(self, p, pitch, c0, c1):
        """Absolute channels in [c0, c1) that are padding in some Act viewing (p, pitch) and real in none."""
        pad, real = set(), set()
        for a in self.acts.get((p, pitch), ()):
            for q, m in enumerate(a.chanmap):
                (real if m >= 0 else pad).add(a.c_off + q)
        return sorted(c for c in pad - real if c0 <= c < c1)


# ------------------------------------------------------------------------------------------------------------ helpers
def _f32(v):
    return torch.tensor(v, dtype=torch.float32)


def lerp_axis(n_in, n_out, shift=0):
    """Legacy-bilinear weights [n_out, n_in] (fp64 from the fp32 position d * fp32(n_in / n_out)) and the 0/1 matrix of the corners read.
    shift: source index off by `shift` (negative control)."""
    step = _f32(n_in) / _f32(n_out)
    s = torch.arange(n_out, dtype=torch.float32) * step
    lo = torch.floor(s)
    f = (s - lo).double()
    lo = (lo.long() + shift).clamp(0, n_in - 1)
    hi = torch.clamp(lo + 1, max=n_in - 1)
    d = torch.arange(n_out)
    M = torch.zeros(n_out, n_in, dtype=torch.float64)
    M.index_put_((d, lo), 1 - f, accumulate=True)
    M.index_put_((d, hi), f, accumulate=True)
    I = torch.zeros(n_out, n_in, dtype=torch.float64)
    I[d, lo] = 1
    I[d, hi] = 1
    return M.cuda(), I.cuda()


def nn2x_axis(n):
    """Nearest x2 (align_corners) one-hot [2n, n]: source min(roundf(d * fp32((n-1)/(2n-1))), n-1)."""
    scale = _f32(n - 1) / _f32(2 * n - 1)
    v = (torch.arange(2 * n, dtype=torch.float32) * scale).double()
    assert not bool(((v - torch.floor(v)) == 0.5).any()), 'roundf tie'
    idx = torch.floor(v + 0.5).long().clamp(max=n - 1)
    M = torch.zeros(2 * n, n, dtype=torch.float64)
    M[torch.arange(2 * n), idx] = 1
    return M.cuda()


def apply2(My, Mx, x):
    """x [N, H, W, C] -> [N, OH, OW, C] with My [OH, H], Mx [OW, W]."""
    return torch.einsum('pw,nowc->nopc', Mx, torch.einsum('oh,nhwc->nowc', My, x))


def apply2_t(My, Mx, d):
    """Transpose of apply2: d [N, OH, OW, C] -> [N, H, W, C]."""
    return torch.einsum('pw,nhpc->nhwc', Mx, torch.einsum('oh,nopc->nhpc', My, d))


def terms2(My, Mx):
    """Nonzero weights of each source element of the transpose, [1, H, W, 1]."""
    ty, tx = (My != 0).sum(0).double(), (Mx != 0).sum(0).double()
    return (ty[:, None] * tx[None, :])[None, :, :, None]


def ratio(got, ref, bound):
    """max |got - ref| / (bound + FLOOR); inf when got holds a non-finite value."""
    got = got.double()
    if not torch.isfinite(got).all():
        return float('inf')
    if got.numel() == 0:
        return 0.0
    return float(((got - ref).abs() / (bound + FLOOR)).max())


def exact(got, ref):
    """0 when got equals ref (after rounding ref to got's dtype) bit for bit, else max |got - ref| / FLOOR (or inf)."""
    r = ref.to(got.dtype)
    if torch.equal(got, r) or (got.numel() == 0):
        return 0.0
    d = (got.double() - r.double()).abs()
    return float('inf') if not torch.isfinite(d).all() else max(float(d.max()) / FLOOR, 1e30)


def _bound(ref, S, gamma, e_out, delta=0.0):
    return e_out * ref.abs() + gamma * S + delta


def _tile(got):
    """Copy of a bf16 result [..., H, W, C] with one 16 x 8 tile of one channel (at the largest value) scaled by 1 + 2^-5."""
    g = got.double().clone()
    flat = g.reshape(-1, *g.shape[-3:])
    n, h, x, c = [int(v) for v in torch.unravel_index(flat.abs().argmax(), flat.shape)]
    flat[n, h // 16 * 16:h // 16 * 16 + 16, x // 8 * 8:x // 8 * 8 + 8, c] *= 1 + 2 ** -5
    return flat.view(g.shape)


def _shift(t, dy, dx):
    """out[:, y, x] = t[:, y + dy, x + dx], zero outside."""
    o = torch.zeros_like(t)
    h, w = t.shape[1], t.shape[2]
    ys, ye, xs, xe = max(0, -dy), min(h, h - dy), max(0, -dx), min(w, w - dx)
    if ys < ye and xs < xe:
        o[:, ys:ye, xs:xe] = t[:, ys + dy:ye + dy, xs + dx:xe + dx]
    return o


def _disps(R):
    return [(dy, dx) for dy in range(-R, R + 1) for dx in range(-R, R + 1)]


def _corr(A, Bm, R):
    """[..., ND]: sum_c A[p, c] Bm[p + d, c] (zero outside)."""
    return torch.stack([(A * _shift(Bm, dy, dx)).sum(-1) for dy, dx in _disps(R)], -1)


# ------------------------------------------------------------------------------------------------------------ warp geometry
class _Warp(object):
    """The warped map of c2 (fp64) and what the bounds need, for cis_warp_costvol and its backward."""

    def __init__(self, c2, flow, fs, fs_scale=1.0):
        B, h, w, C = c2.shape
        self.c2 = c2
        if flow is None:
            self.flow = None
            self.W, self.Werr = c2, torch.zeros_like(c2)
            return
        self.flow = flow
        fs = float(_f32(fs)) * fs_scale
        f = flow.double()
        gy = torch.arange(h, dtype=torch.float64, device=c2.device).view(1, h, 1)
        gx = torch.arange(w, dtype=torch.float64, device=c2.device).view(1, 1, w)
        self.fs = fs
        qy, qx = gy - fs * f[..., 0], gx - fs * f[..., 1]
        self.eps_y = U23 * (qy.abs() + (fs * f[..., 0]).abs())
        self.eps_x = U23 * (qx.abs() + (fs * f[..., 1]).abs())
        ly = torch.floor(qy).clamp(0, h - 2)
        lx = torch.floor(qx).clamp(0, w - 2)
        self.ay, self.ax = (qy - ly).clamp(0, 1), (qx - lx).clamp(0, 1)
        self.pass_y = ((qy - ly) >= 0) & ((qy - ly) <= 1)
        self.pass_x = ((qx - lx) >= 0) & ((qx - lx) <= 1)
        # within eps of an integer: the floor, the clamps and the pass flags may go either way
        self.amb_pos = ((qy - torch.round(qy)).abs() <= self.eps_y) | ((qx - torch.round(qx)).abs() <= self.eps_x)
        self.ly, self.lx = ly.long(), lx.long()
        bidx = torch.arange(B, device=c2.device).view(B, 1, 1)
        self.bidx = bidx
        flat = c2.reshape(B * h * w, C)

        def at(dy, dx):
            yy = (self.ly + dy).clamp(0, h - 1)
            xx = (self.lx + dx).clamp(0, w - 1)
            return flat.index_select(0, ((bidx * h + yy) * w + xx).reshape(-1)).view(B, h, w, C)
        self.tl, self.tr, self.bl, self.br = at(0, 0), at(0, 1), at(1, 0), at(1, 1)
        ay, ax = self.ay[..., None], self.ax[..., None]
        self.t = (1 - ax) * self.tl + ax * self.tr
        self.bo = (1 - ax) * self.bl + ax * self.br
        self.W = (1 - ay) * self.t + ay * self.bo
        self.Sc = self.tl.abs() + self.tr.abs() + self.bl.abs() + self.br.abs()
        # M: max |c2| over rows ly-1 .. ly+2, columns lx-1 .. lx+2
        a = c2.abs().permute(0, 3, 1, 2)
        mp = F.max_pool2d(F.pad(a, (1, 2, 1, 2)), 4, stride=1).permute(0, 2, 3, 1).contiguous()
        self.M = mp.reshape(B * h * w, C).index_select(0, ((bidx * h + self.ly) * w + self.lx).reshape(-1)).view(B, h, w, C)
        self.Werr = G_LERP * self.Sc + (self.eps_y + self.eps_x)[..., None] * 2 * self.M

    def scatter(self, v, weights=True):
        """Bilinear scatter of v [B, h, w, C] (the transpose of the warp) -> [B, h, w, C]."""
        B, h, w, C = v.shape
        out = torch.zeros(B * h * w, C, dtype=torch.float64, device=v.device)
        ay, ax = self.ay[..., None], self.ax[..., None]
        for dy, dx, wt in ((0, 0, (1 - ay) * (1 - ax)), (0, 1, (1 - ay) * ax), (1, 0, ay * (1 - ax)), (1, 1, ay * ax)):
            idx = ((self.bidx * h + self.ly + dy) * w + self.lx + dx).reshape(-1)
            out.index_add_(0, idx, (v * (wt if weights else 1.0)).reshape(-1, C))
        return out.view(B, h, w, C)

    def spread(self, v):
        """v [B, h, w, C] added to all 16 pixels of the 4 x 4 neighbourhood of each cell (clamped)."""
        B, h, w, C = v.shape
        out = torch.zeros(B * h * w, C, dtype=torch.float64, device=v.device)
        for dy in range(-1, 3):
            for dx in range(-1, 3):
                idx = ((self.bidx * h + (self.ly + dy).clamp(0, h - 1)) * w + (self.lx + dx).clamp(0, w - 1)).reshape(-1)
                out.index_add_(0, idx, v.reshape(-1, C))
        return out.view(B, h, w, C)


# ------------------------------------------------------------------------------------------------------------ unsupervised loss
U24 = 2.0 ** -24


def _unsup_sample(img, flow):
    """dense_image_warp's sample of img [N,H,W,C] at q = p - flow (fp64, exact alphas): val, abs = sum of the four |corners|, the
    derivative factors cy = bot - top and cx = ay (br - bl) + (1 - ay)(tr - tl), and the pass flags of the alphas."""
    import unsup_flow_loss_ref as UR
    N, H, W, C = img.shape
    qy, qx = UR.sample_points(flow)

    def prep(q, size):
        fl = torch.clamp(torch.floor(q), 0.0, float(size - 2))
        r = q - fl
        return fl.long(), torch.clamp(r, 0.0, 1.0).unsqueeze(-1), (r >= 0) & (r <= 1)
    fy, ay, py = prep(qy, H)
    fx, ax, px = prep(qx, W)
    flat = img.reshape(N, H * W, C)

    def at(yy, xx):
        return torch.gather(flat, 1, (yy * W + xx).reshape(N, H * W, 1).expand(-1, -1, C)).reshape(N, H, W, C)
    tl, tr, bl, br = at(fy, fx), at(fy, fx + 1), at(fy + 1, fx), at(fy + 1, fx + 1)
    top, bot = tl + ax * (tr - tl), bl + ax * (br - bl)
    return dict(val=top + ay * (bot - top), abs=tl.abs() + tr.abs() + bl.abs() + br.abs(), cy=bot - top,
                cx=ay * (br - bl) + (1 - ay) * (tr - tl), pass_y=py, pass_x=px)


def _tsoft(v):
    return v / torch.sqrt(0.81 + v * v)


def _tsoft_slope(v):
    """max of |t'| over |v'| >= |v| (t' = 0.81 / (0.81 + v^2)^1.5 falls with |v|)."""
    return 0.81 / (0.81 + v * v) ** 1.5


def _census_bound(gS, tw):
    """c of unsup_flow_loss_ref.census and the bound e on the kernel's fp32 c: gray levels of S rounded to fp32 (2^-24 each), T~ read
    as is, differences rounded, t(v) = v rsqrtf(0.81 + v^2) within 8 2^-24 |t| (rsqrtf 2 ulp, three roundings, the constant 0.81f),
    the difference e = t_S - t_T carried through phi(e) = e^2 / (0.1 + e^2) by its largest slope on [|e| - e_e, |e| + e_e], phi's own
    roundings 8 2^-24 phi, and the 48-term fp32 sum (48 2^-23 c)."""
    import unsup_flow_loss_ref as UR
    c, e = torch.zeros_like(tw), torch.zeros_like(tw)
    xs = (0.1 / 3) ** 0.5                                 # phi' = 0.2 x / (0.1 + x^2)^2 peaks there
    for dy in range(-3, 4):
        for dx in range(-3, 4):
            if dy == 0 and dx == 0:
                continue
            s2, ins = UR._shift(gS, dy, dx)
            t2, _ = UR._shift(tw, dy, dx)
            vS, vT = s2 - gS, t2 - tw
            e_vS, e_vT = U24 * (s2.abs() + gS.abs() + vS.abs()), U24 * vT.abs()
            tS, tT = _tsoft(vS), _tsoft(vT)
            e_d = (_tsoft_slope(torch.clamp(vS.abs() - e_vS, min=0)) * e_vS + 8 * U24 * tS.abs() +
                   _tsoft_slope(torch.clamp(vT.abs() - e_vT, min=0)) * e_vT + 8 * U24 * tT.abs())
            d = tS - tT
            e_d = e_d + U24 * d.abs()
            x = torch.clamp(torch.full_like(d, xs), min=torch.clamp(d.abs() - e_d, min=0), max=d.abs() + e_d)
            phi = d * d / (0.1 + d * d)
            c = c + ins * phi
            e = e + ins * (0.2 * x / (0.1 + x * x) ** 2 * e_d + 8 * U24 * phi)
    return dict(c=c, e=e + 48 * U23 * c)


def _unsup_smooth_terms(fd, S):
    """Per pixel of the 2B directions: val = sum_a w_a s_a (the kernel's per-pixel smoothness term) and err, its bound: w_a within
    rel_w (fp32 differences and sums of the frame, the 1/3f and -10 products, expf 2 ulp), and where |l_c| is within 2^-50 (|a| + 2|b|
    + |c|) of the ROUNDING threshold (the double second difference may land on either side) w |l_c| more.  Per axis, for the backward's
    gather: X = w sign(l) per centre, A = w, Rw = w rel_w, Z = w at centres whose sign is ambiguous ([N,H,W,2]; 0 where no centre)."""
    import unsup_flow_loss_ref as UR
    N, H, W, _ = fd.shape
    val, err = torch.zeros(N, H, W, dtype=fd.dtype, device=fd.device), torch.zeros(N, H, W, dtype=fd.dtype, device=fd.device)
    axes = []
    for dim in (1, 2):
        n = fd.shape[dim]
        a, b, c = fd.narrow(dim, 2, n - 2), fd.narrow(dim, 1, n - 2), fd.narrow(dim, 0, n - 2)
        l = a - 2 * b + c
        mag = a.abs() + 2 * b.abs() + c.abs()
        amb = (l.abs() - UR.ROUNDING * mag).abs() <= 2.0 ** -50 * mag
        lz = UR.second_difference(a, b, c)
        e3 = (S.narrow(dim, 2, n - 2) - S.narrow(dim, 0, n - 2)).abs().sum(-1)
        w = torch.exp(-10.0 * (e3 / 3) / 2)
        rel_w = 5 * (e3 / 3) * 8 * U24 + 3 * U23
        s = lz.abs().sum(-1)
        v_in = w * s
        e_in = rel_w * v_in + w * (amb * l.abs()).sum(-1) + 2.0 ** -50 * v_in
        pad = [0, 0] * (2 - dim) + [1, 1]
        val = val + F.pad(v_in, pad)
        err = err + F.pad(e_in, pad)
        pad4 = [0, 0] + pad
        X = F.pad(w.unsqueeze(-1) * torch.sign(lz), pad4)
        A = F.pad(w.unsqueeze(-1) * torch.ones_like(lz), pad4)
        Rw = F.pad((w * rel_w).unsqueeze(-1) * torch.ones_like(lz), pad4)
        Z = F.pad(w.unsqueeze(-1) * amb, pad4)
        axes.append((dim, X, A, Rw, Z))
    return dict(val=val, err=err, axes=axes)


def _stencil(X, dim, centre):
    """out[r] = X[r + e] + X[r - e] + centre X[r] along dim (0 outside)."""
    n = X.shape[dim]
    out = centre * X
    z = torch.zeros_like(X.narrow(dim, 0, 1))
    out = out + torch.cat([X.narrow(dim, 1, n - 1), z], dim) + torch.cat([z, X.narrow(dim, 0, n - 1)], dim)
    return out


def unsup_bwd_gather(flow, img1, img2, warped, coef, w_photo, w_smooth, bounds=False):
    """cis_unsup_flow_loss_bwd restated as an explicit fp64 gather on any device: the census term folded into one sweep of each pixel's
    own 7x7 window, dT~(r) = -w_photo sum_d (k(r+d) + k(r)) h(r, r+d), h = d/du of phi(t_S - t(u)) at u = T~(r+d) - T~(r), chained
    through dense_image_warp's dflow rule at r's own sample point; plus w_smooth times the 5-point gather of w sign(l) from the centres
    r - e_a (x1), r (x-2), r + e_a (x1).  flow [2B,H,W,2], frames [B,H,W,3], warped / coef [2B,H,W] (the forward's T~ and M psi'(c)).
    -> dict(ref, photo (the census part alone), smooth) and with bounds=True err, the bound on the kernel's fp32 result."""
    import unsup_flow_loss_ref as UR
    S, T = UR.directions(img1, img2)
    gS = UR.gray(S)
    G, eG, SG = torch.zeros_like(warped), torch.zeros_like(warped), torch.zeros_like(warped)
    for dy in range(-3, 4):
        for dx in range(-3, 4):
            if dy == 0 and dx == 0:
                continue
            s2, ins = UR._shift(gS, dy, dx)
            t2, _ = UR._shift(warped, dy, dx)
            k2, _ = UR._shift(coef, dy, dx)
            vS, u = s2 - gS, t2 - warped
            iu = 1 / torch.sqrt(0.81 + u * u)
            d = _tsoft(vS) - u * iu
            hh = -0.2 * d / (0.1 + d * d) ** 2 * 0.81 * iu ** 3
            term = ins * (k2 + coef) * hh
            G = G + term
            if bounds:
                # |d(-0.2 d / (0.1 + d^2)^2) / dd| <= 0.2 (0.1 + 3x) / (0.1 + x)^3, x = d^2, which falls with x; ~33 fp32 roundings
                # (rsqrtf 2 ulp, iu^3, den^2, the products, the constants 0.2f and 0.81f, k2 + k) on the term itself
                e_vS, e_u = U24 * (s2.abs() + gS.abs() + vS.abs()), U24 * u.abs()
                e_d = (_tsoft_slope(torch.clamp(vS.abs() - e_vS, min=0)) * e_vS + 8 * U24 * _tsoft(vS).abs() +
                       _tsoft_slope(torch.clamp(u.abs() - e_u, min=0)) * e_u + 8 * U24 * (u * iu).abs())
                e_d = e_d + U24 * d.abs()
                x = torch.clamp(d.abs() - e_d, min=0) ** 2
                slope = 0.2 * (0.1 + 3 * x) / (0.1 + x) ** 3 * 0.81 * iu ** 3
                eG = eG + ins * (k2 + coef).abs() * (slope * e_d + 33 * U24 * hh.abs())
                SG = SG + term.abs()
    dtw = -G * w_photo
    st = _unsup_sample(UR.gray(T).unsqueeze(-1), flow)
    cy, cx = st['cy'][..., 0], st['cx'][..., 0]
    photo = torch.stack([torch.where(st['pass_y'], -dtw * cy, torch.zeros_like(cy)), torch.where(st['pass_x'], -dtw * cx, torch.zeros_like(cx))], -1)
    sm = _unsup_smooth_terms(flow, S)
    smooth = torch.zeros_like(flow)
    absw, relw, ambw = torch.zeros_like(flow), torch.zeros_like(flow), torch.zeros_like(flow)
    for dim, X, A, Rw, Z in sm['axes']:
        smooth = smooth + _stencil(X, dim, -2.0)
        absw = absw + _stencil(A, dim, 2.0)
        relw = relw + _stencil(Rw, dim, 2.0)
        ambw = ambw + _stencil(Z, dim, 2.0)
    ref = photo + w_smooth * smooth
    out = dict(ref=ref, photo=photo, smooth=smooth)
    if bounds:
        e_dtw = w_photo * (eG + 48 * U23 * SG) + U24 * dtw.abs()
        e_chain = 2.0 ** -20 * st['abs'][..., 0]              # fp32 gray corners and alphas, the lerps
        pas = torch.stack([st['pass_y'], st['pass_x']], -1)
        e_photo = pas * ((dtw.abs() * e_chain).unsqueeze(-1) + torch.stack([cy, cx], -1).abs() * e_dtw.unsqueeze(-1) + U24 * photo.abs())
        # the weights' own error, the 6-term fp32 sum, the ambiguous signs
        e_sm = w_smooth * (relw + 6 * U23 * absw + ambw) + U24 * (w_smooth * smooth).abs()
        out['err'] = e_photo + e_sm + U23 * ref.abs()
    return out


# ------------------------------------------------------------------------------------------------------------ the checker
class Glue(object):
    """Per-launch checks of the glue entry points.  results[label] = bound ratios; counts[entry point] = launches checked; failures =
    messages; controls[name] = negative-control ratio (> 1: rejected), when made with controls=True."""

    def __init__(self, controls=False):
        self.mem = Mem()
        self.results = collections.defaultdict(list)
        self.counts = collections.Counter()
        self.failures = []
        self.controls = {} if controls else None
        self.first_nonfinite = None       # (plan, index, entry point) of the first launch that read a non-finite operand
        self.where = ('', 0)
        self.colpart = collections.defaultdict(list)    # storage offset intervals the partial-sum launches of this plan wrote

    @staticmethod
    def owns(name):
        return name in ARGS

    def start_plan(self, name):
        self.where = (name, 0)
        self.colpart.clear()

    # ---- driver
    def before(self, op, index=0):
        self.where = (self.where[0], index)
        a = decode(op)
        ctx = getattr(self, '_pre_' + op[2][4:])(a)
        ctx['snap'] = {}
        for win in ctx['dests']:
            t, off = self.mem.storage(win[0])
            key = t.untyped_storage().data_ptr()
            if key not in ctx['snap']:
                ctx['snap'][key] = (t, t.clone())
        reads = ctx.pop('reads', [])
        if self.first_nonfinite is None and any(not bool(torch.isfinite(r).all()) for r in reads):
            self.first_nonfinite = (self.where[0], index, op[2])
        return ctx

    def after(self, op, ctx):
        a = decode(op)
        getattr(self, '_post_' + op[2][4:])(a, ctx)
        self.counts[op[2]] += 1
        self._stray(op[2], ctx)

    def _rec(self, label, what, r):
        self.results[label].append(r)
        if not r <= 1.0:
            self.failures.append('%s launch %d %s: %s bound ratio %.3g' % (self.where[0], self.where[1], label, what, r))

    def _control(self, name, r):
        if self.controls is not None and name not in self.controls:
            self.controls[name] = r

    def _stray(self, name, ctx):
        """Outside the windows of ctx['dests'] = [(ptr, dtype, rows, pitch, c0, c1)], every byte unchanged; padding channels 0."""
        groups = collections.defaultdict(list)
        for win in ctx['dests']:
            t, off = self.mem.storage(win[0])
            groups[t.untyped_storage().data_ptr()].append((off,) + tuple(win))
        for key, wins in groups.items():
            now, old = ctx['snap'][key]
            masked = now.clone()
            for off, p, dtype, rows, pitch, c0, c1 in wins:
                n = rows * pitch * dtype.itemsize
                masked[off:off + n].view(dtype).view(rows, pitch)[:, c0:c1] = old[off:off + n].view(dtype).view(rows, pitch)[:, c0:c1]
            if not torch.equal(masked, old):
                diff = (masked != old).nonzero()
                self.failures.append('%s launch %d %s: stray write at byte %d of its destination storage'
                                     % (self.where[0], self.where[1], name, int(diff[0])))
            for off, p, dtype, rows, pitch, c0, c1 in wins:
                if dtype != torch.bfloat16:
                    continue
                pads = self.mem.pads(p, pitch, c0, c1)
                if pads:
                    v = now[off:off + rows * pitch * 2].view(dtype).view(rows, pitch)[:, pads]
                    if not bool((v == 0).all()):
                        self.failures.append('%s launch %d %s: padding channels %s not zero' % (self.where[0], self.where[1], name, pads))

    def _bf(self, p, rows, pitch):
        return self.mem.view(p, torch.bfloat16, (rows, pitch))

    # ---- cis_zero
    def _pre_zero(self, a):
        n = a['nbytes']
        return dict(dests=[(a['ptr'], torch.uint8, 1, n, 0, n)])

    def _post_zero(self, a, ctx):
        got = self.mem.view(a['ptr'], torch.uint8, (a['nbytes'],))
        self._rec('cis_zero', 'zero fill', 0.0 if bool((got == 0).all()) else float('inf'))

    # ---- cis_pack_f32_to_bf16
    def _pre_pack_f32_to_bf16(self, a):
        n, C = a['npix'], a['C']
        src = self.mem.view(a['src'], torch.float32, (n, C)).clone()
        ref = torch.zeros(n, 8, dtype=torch.float32, device='cuda')
        ref[:, :C] = src + _f32(a['offset']).cuda()
        return dict(ref=ref.to(torch.bfloat16), reads=[src], dests=[(a['dst'], torch.bfloat16, n, a['dp'], a['dc'], a['dc'] + 8)])

    def _post_pack_f32_to_bf16(self, a, ctx):
        got = self._bf(a['dst'], a['npix'], a['dp'])[:, a['dc']:a['dc'] + 8]
        self._rec('cis_pack_f32_to_bf16', 'packed input', exact(got, ctx['ref']))

    # ---- cis_cast_bf16_to_f32
    def _pre_cast_bf16_to_f32(self, a):
        n, C = a['npix'], a['C']
        src = self._bf(a['src'], n, a['pitch'])[:, a['coff']:a['coff'] + C].clone()
        return dict(ref=src.float(), reads=[src], dests=[(a['dst'], torch.float32, n, C, 0, C)])

    def _post_cast_bf16_to_f32(self, a, ctx):
        got = self.mem.view(a['dst'], torch.float32, (a['npix'], a['C']))
        self._rec('cis_cast_bf16_to_f32', 'cast', exact(got, ctx['ref']))

    # ---- cis_parity_split_bf16
    def _pre_parity_split_bf16(self, a):
        N, H, W, C, sp, sc = a['N'], a['H'], a['W'], a['C'], a['sp'], a['sc']
        src = self.mem.view(a['src'], torch.bfloat16, (N, 2 * H, 2 * W, sp))[..., sc:sc + C].clone()
        ref = torch.zeros(4, N, H, W, 8, dtype=torch.bfloat16, device='cuda')
        for q in range(4):
            ref[q, ..., :C] = src[:, q >> 1::2, q & 1::2]
        return dict(ref=ref.view(4 * N * H * W, 8), reads=[src], dests=[(a['dst'], torch.bfloat16, 4 * N * H * W, a['dp'], 0, 8)])

    def _post_parity_split_bf16(self, a, ctx):
        got = self._bf(a['dst'], 4 * a['N'] * a['H'] * a['W'], a['dp'])[:, :8]
        self._rec('cis_parity_split_bf16', 'parity planes', exact(got, ctx['ref']))

    # ---- cis_upsample_nn2x and its transpose
    def _pre_upsample_nn2x(self, a):
        N, H, W, P = a['N'], a['H'], a['W'], a['pitch']
        src = self.mem.view(a['src'], torch.bfloat16, (N, H, W, P)).clone()
        ref = apply2(nn2x_axis(H), nn2x_axis(W), src.double())
        return dict(ref=ref, reads=[src], dests=[(a['dst'], torch.bfloat16, N * 4 * H * W, P, 0, P)])

    def _post_upsample_nn2x(self, a, ctx):
        N, H, W, P = a['N'], a['H'], a['W'], a['pitch']
        got = self.mem.view(a['dst'], torch.bfloat16, (N, 2 * H, 2 * W, P))
        self._rec('cis_upsample_nn2x', 'nearest x2', exact(got, ctx['ref']))

    def _pre_upsample_nn2x_bwd(self, a):
        N, H, W, P = a['N'], a['H'], a['W'], a['pitch']
        dd = self.mem.view(a['dd'], torch.bfloat16, (N, 2 * H, 2 * W, P)).clone()
        My, Mx = nn2x_axis(H), nn2x_axis(W)
        ref, S = apply2_t(My, Mx, dd.double()), apply2_t(My, Mx, dd.double().abs())
        if a['acc']:
            old = self.mem.view(a['ds'], torch.bfloat16, (N, H, W, P)).double()
            ref, S = ref + old, S + old.abs()
        gamma = (terms2(My, Mx) + 1) * U23
        return dict(ref=ref, S=S, gamma=gamma, reads=[dd], dests=[(a['ds'], torch.bfloat16, N * H * W, P, 0, P)])

    def _post_upsample_nn2x_bwd(self, a, ctx):
        got = self.mem.view(a['ds'], torch.bfloat16, (a['N'], a['H'], a['W'], a['pitch']))
        b = _bound(ctx['ref'], ctx['S'], ctx['gamma'] * (1 + 2 ** -7), E_BF16)
        self._rec('cis_upsample_nn2x_bwd', 'nearest x2 transpose', ratio(got, ctx['ref'], b))

    # ---- legacy bilinear resizes
    def _pre_resize_bilinear_f32(self, a):
        N, H, W, C, OH, OW = a['N'], a['H'], a['W'], a['C'], a['OH'], a['OW']
        src = self.mem.view(a['src'], torch.float32, (N, H, W, C)).clone()
        (My, Iy), (Mx, Ix) = lerp_axis(H, OH), lerp_axis(W, OW)
        sc = float(_f32(a['scale']))
        x = src.double()
        ctx = dict(ref=apply2(My, Mx, x) * sc, S=apply2(Iy, Ix, x.abs()) * abs(sc), reads=[src],
                   dests=[(a['dst'], torch.float32, N * OH * OW, C, 0, C)])
        if self.controls is not None and 'resize.row_off_by_one' not in self.controls:
            ctx['bad'] = apply2(lerp_axis(H, OH, shift=1)[0], Mx, x) * sc
        return ctx

    def _post_resize_bilinear_f32(self, a, ctx):
        got = self.mem.view(a['dst'], torch.float32, (a['N'], a['OH'], a['OW'], a['C']))
        b = _bound(ctx['ref'], ctx['S'], G_LERP, 0.0)
        self._rec('cis_resize_bilinear_f32', 'fp32 resize', ratio(got, ctx['ref'], b))
        if 'bad' in ctx:
            self._control('resize.row_off_by_one', ratio(got, ctx['bad'], b))

    def _pre_resize_bilinear_bf16(self, a):
        N, H, W, OH, OW, ch = a['N'], a['H'], a['W'], a['OH'], a['OW'], a['chunks'] * 8
        src = self.mem.view(a['src'], torch.bfloat16, (N, H, W, a['sp']))[..., a['sc']:a['sc'] + ch].clone()
        (My, Iy), (Mx, Ix) = lerp_axis(H, OH), lerp_axis(W, OW)
        x = src.double()
        return dict(ref=apply2(My, Mx, x), S=apply2(Iy, Ix, x.abs()), reads=[src],
                    dests=[(a['dst'], torch.bfloat16, N * OH * OW, a['dp'], a['dc'], a['dc'] + ch)])

    def _post_resize_bilinear_bf16(self, a, ctx):
        ch = a['chunks'] * 8
        got = self.mem.view(a['dst'], torch.bfloat16, (a['N'], a['OH'], a['OW'], a['dp']))[..., a['dc']:a['dc'] + ch]
        b = _bound(ctx['ref'], ctx['S'], G_LERP * (1 + 2 ** -7), E_BF16)
        self._rec('cis_resize_bilinear_bf16', 'bf16 resize', ratio(got, ctx['ref'], b))
        self._control('tile.cis_resize_bilinear_bf16', ratio(_tile(got), ctx['ref'], b))

    def _pre_resize_bilinear_bf16_bwd(self, a):
        N, H, W, OH, OW, ch = a['N'], a['H'], a['W'], a['OH'], a['OW'], a['chunks'] * 8
        dd = self.mem.view(a['dd'], torch.bfloat16, (N, OH, OW, a['dp']))[..., a['dc']:a['dc'] + ch].clone()
        (My, _), (Mx, _) = lerp_axis(H, OH), lerp_axis(W, OW)
        ref, S = apply2_t(My, Mx, dd.double()), apply2_t(My, Mx, dd.double().abs())
        if a['acc']:
            old = self.mem.view(a['ds'], torch.bfloat16, (N, H, W, a['sp']))[..., a['sc']:a['sc'] + ch].double()
            ref, S = ref + old, S + old.abs()
        return dict(ref=ref, S=S, gamma=(terms2(My, Mx) + 1) * U23, reads=[dd],
                    dests=[(a['ds'], torch.bfloat16, N * H * W, a['sp'], a['sc'], a['sc'] + ch)])

    def _post_resize_bilinear_bf16_bwd(self, a, ctx):
        ch = a['chunks'] * 8
        got = self.mem.view(a['ds'], torch.bfloat16, (a['N'], a['H'], a['W'], a['sp']))[..., a['sc']:a['sc'] + ch]
        b = _bound(ctx['ref'], ctx['S'], ctx['gamma'] * (1 + 2 ** -7), E_BF16)
        self._rec('cis_resize_bilinear_bf16_bwd', 'bf16 resize transpose', ratio(got, ctx['ref'], b))

    def _pre_resize_f32_bwd_to_bf16_scaled(self, a):
        N, OH, OW, C, H, W = a['N'], a['OH'], a['OW'], a['C'], a['H'], a['W']
        dd = self.mem.view(a['dd'], torch.float32, (N, OH, OW, C)).clone()
        (My, _), (Mx, _) = lerp_axis(H, OH), lerp_axis(W, OW)
        sc = float(_f32(a['scale']))
        ref = torch.zeros(N, H, W, 8, dtype=torch.float64, device='cuda')
        S = torch.zeros_like(ref)
        ref[..., :C] = apply2_t(My, Mx, dd.double()) * sc
        S[..., :C] = apply2_t(My, Mx, dd.double().abs()) * abs(sc)
        # + 1 more rounding: the final scale multiply
        return dict(ref=ref, S=S, gamma=(terms2(My, Mx) + 2) * U23, reads=[dd], dests=[(a['ds'], torch.bfloat16, N * H * W, a['sp'], 0, 8)])

    def _post_resize_f32_bwd_to_bf16_scaled(self, a, ctx):
        got = self.mem.view(a['ds'], torch.bfloat16, (a['N'], a['H'], a['W'], a['sp']))[..., :8]
        b = _bound(ctx['ref'], ctx['S'], ctx['gamma'] * (1 + 2 ** -7), E_BF16)
        self._rec('cis_resize_f32_bwd_to_bf16_scaled', 'scaled resize transpose', ratio(got, ctx['ref'], b))

    # ---- fused resize + concat and its transpose
    @staticmethod
    def _rc_kind(H, W, OH, OW):
        return 'same' if (H, W) == (OH, OW) else 'x2' if (OH, OW) == (2 * H, 2 * W) else 'generic'

    def _pre_resize_concat_bf16(self, a):
        N, H, W, OH, OW = a['N'], a['H'], a['W'], a['OH'], a['OW']
        xs = []
        for s in list(a['srcs'])[:a['nsrc']]:
            rows = s.n_mod if s.n_mod else N
            x = self.mem.view(s.ptr, torch.bfloat16, (rows, H, W, s.pitch))[..., s.c_off:s.c_off + 8 * s.chunks]
            if s.n_mod:
                x = x[torch.arange(N, device=x.device) % s.n_mod]
            xs.append(x)
        X = torch.cat(xs, 3).clone()
        kind = self._rc_kind(H, W, OH, OW)
        ctx = dict(kind=kind, tc=X.shape[3], reads=[X], dests=[(a['dst'], torch.bfloat16, N * OH * OW, a['dp'], a['dc'], a['dc'] + X.shape[3])])
        if kind == 'same':
            ctx['ref'] = X
        else:
            (My, Iy), (Mx, Ix) = lerp_axis(H, OH), lerp_axis(W, OW)
            x = X.double()
            ctx['ref'], ctx['S'] = apply2(My, Mx, x), apply2(Iy, Ix, x.abs())
            if self.controls is not None and 'resize.row_off_by_one' not in self.controls:
                ctx['bad'] = apply2(lerp_axis(H, OH, shift=1)[0], Mx, x)
        return ctx

    def _post_resize_concat_bf16(self, a, ctx):
        got = self.mem.view(a['dst'], torch.bfloat16, (a['N'], a['OH'], a['OW'], a['dp']))[..., a['dc']:a['dc'] + ctx['tc']]
        label = 'cis_resize_concat_bf16.' + ctx['kind']
        if ctx['kind'] == 'same':
            return self._rec(label, 'concat', exact(got, ctx['ref']))
        b = _bound(ctx['ref'], ctx['S'], G_LERP * (1 + 2 ** -7), E_BF16)
        self._rec(label, 'resize-concat', ratio(got, ctx['ref'], b))
        if 'bad' in ctx:
            self._control('resize.row_off_by_one', ratio(got, ctx['bad'], b))
        self._control('tile.' + label, ratio(_tile(got), ctx['ref'], b))

    def _pre_resize_concat_bf16_bwd(self, a):
        N, OH, OW, H, W = a['N'], a['OH'], a['OW'], a['H'], a['W']
        kind = self._rc_kind(H, W, OH, OW)
        if kind == 'same':
            My = Mx = None
        else:
            (My, _), (Mx, _) = lerp_axis(H, OH), lerp_axis(W, OW)
        dd_all = self.mem.view(a['dd'], torch.bfloat16, (N, OH, OW, a['dp']))
        per, dests, reads, off = [], [], [], a['dc']
        for i, s in enumerate(list(a['grads'])[:a['nsrc']]):
            ch = 8 * s.chunks
            want, acc = int(a['want'][i]), int(a['acc'][i])
            if want:
                dd = dd_all[..., off:off + ch].clone().double()
                reads.append(dd)
                rows = s.n_mod if s.n_mod else N
                reps = N // rows
                parts = [dd[r * rows:(r + 1) * rows] for r in range(reps)]
                tr = (lambda v: v) if kind == 'same' else (lambda v: apply2_t(My, Mx, v))
                folded = [tr(p) for p in parts]
                ref, S = sum(folded), sum(tr(p.abs()) for p in parts)
                terms = reps * (1.0 if kind == 'same' else terms2(My, Mx))
                old = self.mem.view(s.ptr, torch.bfloat16, (rows, H, W, s.pitch))[..., s.c_off:s.c_off + ch].double()
                ent = dict(i=i, s=s, rows=rows, reps=reps, acc=acc, ref=ref + old if acc else ref, S=S + old.abs() if acc else S,
                           gamma=(terms + 1) * U23, old=old, folded0=folded[0])
                per.append(ent)
                dests.append((s.ptr, torch.bfloat16, rows * H * W, s.pitch, s.c_off, s.c_off + ch))
            off += ch
        return dict(kind=kind, per=per, reads=reads, dests=dests)

    def _post_resize_concat_bf16_bwd(self, a, ctx):
        H, W = a['H'], a['W']
        label = 'cis_resize_concat_bf16_bwd.' + ctx['kind']
        for e in ctx['per']:
            s = e['s']
            got = self.mem.view(s.ptr, torch.bfloat16, (e['rows'], H, W, s.pitch))[..., s.c_off:s.c_off + 8 * s.chunks]
            b = _bound(e['ref'], e['S'], e['gamma'] * (1 + 2 ** -7), E_BF16)
            self._rec(label, 'source %d gradient' % e['i'], ratio(got, e['ref'], b))
            if self.controls is None:
                continue
            if e['reps'] > 1:
                self._control('rc_bwd.fold_dropped', ratio(got, e['folded0'] + (e['old'] if e['acc'] else 0), b))
            if e['acc'] and bool((e['old'] != 0).any()):
                self._control('rc_bwd.overwrite', ratio(got, e['ref'] - e['old'], b))

    # ---- activation derivative, column sums, residual gradients
    def _dact_ref(self, a, nch8, at_y=False):
        n = a['npix']
        g = self._bf(a['g'], n, a['gp'])[:, a['gc']:a['gc'] + nch8].clone()
        y = self._bf(a['y'], n, a['yp'])[:, a['yc']:a['yc'] + nch8].clone()
        u = y.float()
        reads = [g, y]
        if a['res'] and not at_y:
            r = self._bf(a['res'], n, a['rp'])[:, a['rc']:a['rc'] + nch8].clone()
            u = u - r.float()
            reads.append(r)
        alpha = _f32(a['alpha']).cuda()
        d = torch.where(u > 0, torch.ones_like(u), (u + 1) if a['act'] == ACT_ELU else alpha.expand_as(u))
        return (g.float() * d).to(torch.bfloat16), reads

    def _dact_control(self, a, got, ref, nch8):
        if self.controls is None or 'dact.d_at_y' in self.controls or not a['res']:
            return
        bad, _ = self._dact_ref(a, nch8, at_y=True)
        if not torch.equal(bad, ref):         # d(y) and d(y - res) disagree somewhere in this launch
            self.controls['dact.d_at_y'] = exact(got, bad)

    def _pre_dact_mul(self, a):
        nch8 = 8 * a['chunks']
        ref, reads = self._dact_ref(a, nch8)
        ctx = dict(ref=ref, nch8=nch8, reads=reads, dests=[(a['g'], torch.bfloat16, a['npix'], a['gp'], a['gc'], a['gc'] + nch8)])
        if self.controls is not None and a['res'] and 'dact.d_at_y' not in self.controls:
            ctx['bad'] = self._dact_ref(a, nch8, at_y=True)[0]
        return ctx

    def _post_dact_mul(self, a, ctx):
        got = self._bf(a['g'], a['npix'], a['gp'])[:, a['gc']:a['gc'] + ctx['nch8']]
        self._rec('cis_dact_mul', 'activation derivative', exact(got, ctx['ref']))
        if 'bad' in ctx and not torch.equal(ctx['bad'], ctx['ref']):
            self._control('dact.d_at_y', exact(got, ctx['bad']))

    def _colsum_prep(self, a, gref, P):
        n, nch, nblk = a['npix'], a['nch'], a['nblk']
        g = gref[:, :nch].double()
        return dict(cs=g.sum(0), cS=g.abs().sum(0), cgamma=(-(-n // (nblk * P)) + P) * U23)

    def _colsum_check(self, label, a, ctx):
        nblk, nch = a['nblk'], a['nch']
        part = self.mem.view(a['part'], torch.float32, (nblk, nch)).double()
        b = ctx['cgamma'] * ctx['cS']
        self._rec(label, 'column-sum partials', ratio(part.sum(0), ctx['cs'], b))
        # partial rows of one layer's calls are disjoint within a plan (the siamese layers own [call * nblk, (call + 1) * nblk))
        t, off = self.mem.storage(a['part'])
        key, iv = t.untyped_storage().data_ptr(), (off, off + 4 * nblk * nch)
        for o in self.colpart[key]:
            if o[0] < iv[1] and iv[0] < o[1]:
                self.failures.append('%s launch %d %s: partial rows overlap an earlier launch of the plan' % (self.where + (label,)))
        self.colpart[key].append(iv)
        if self.controls is not None and 'colsum.block_dropped' not in self.controls and nblk > 1:
            k = int(part.abs().sum(1).argmax())
            self._control('colsum.block_dropped', ratio(part.sum(0) - part[k], ctx['cs'], b))

    def _pre_dact_colsum(self, a):
        nch8 = 8 * (-(-a['nch'] // 8))
        ref, reads = self._dact_ref(a, nch8)
        ctx = dict(ref=ref, nch8=nch8, reads=reads, dests=[(a['g'], torch.bfloat16, a['npix'], a['gp'], a['gc'], a['gc'] + nch8),
                                                          (a['part'], torch.float32, a['nblk'], a['nch'], 0, a['nch'])])
        ctx.update(self._colsum_prep(a, ref, 256 // (nch8 // 8)))
        if self.controls is not None and a['res'] and 'dact.d_at_y' not in self.controls:
            ctx['bad'] = self._dact_ref(a, nch8, at_y=True)[0]
        return ctx

    def _post_dact_colsum(self, a, ctx):
        got = self._bf(a['g'], a['npix'], a['gp'])[:, a['gc']:a['gc'] + ctx['nch8']]
        self._rec('cis_dact_colsum', 'activation derivative', exact(got, ctx['ref']))
        if 'bad' in ctx and not torch.equal(ctx['bad'], ctx['ref']):
            self._control('dact.d_at_y', exact(got, ctx['bad']))
        self._colsum_check('cis_dact_colsum', a, ctx)

    def _pre_colsum(self, a):
        nch8 = 8 * (-(-a['nch'] // 8))
        g = self._bf(a['g'], a['npix'], a['gp'])[:, a['gc']:a['gc'] + nch8].clone()
        ctx = dict(reads=[g], dests=[(a['part'], torch.float32, a['nblk'], a['nch'], 0, a['nch'])])
        ctx.update(self._colsum_prep(a, g, 256 // (nch8 // 8)))
        return ctx

    def _post_colsum(self, a, ctx):
        self._colsum_check('cis_colsum', a, ctx)

    def _pre_add_slice(self, a):
        n, ch = a['npix'], 8 * a['chunks']
        acc = self._bf(a['dst'], n, a['dp'])[:, a['dc']:a['dc'] + ch].float() if a['acc'] else \
            torch.zeros(n, ch, dtype=torch.float32, device='cuda')
        ctx = dict(ch=ch, dests=[(a['dst'], torch.bfloat16, n, a['dp'], a['dc'], a['dc'] + ch)])
        reads = []
        ref, bad = acc.clone(), torch.zeros_like(acc)
        if a['reps']:
            src = self._bf(a['src'], n * a['reps'], a['sp'])[:, a['sc']:a['sc'] + ch].clone()
            reads.append(src)
            for j in range(a['reps']):                 # the kernel's order: accumulate term first, then the sources
                ref = ref + src[j * n:(j + 1) * n].float()
                bad = bad + src[j * n:(j + 1) * n].float()
            if a['acc']:
                ctx['bad'] = bad.to(torch.bfloat16)
        ctx['ref'], ctx['reads'] = ref.to(torch.bfloat16), reads
        ctx['form'] = 'zero' if not a['reps'] else 'accumulate' if a['acc'] else 'copy'
        return ctx

    def _post_add_slice(self, a, ctx):
        got = self._bf(a['dst'], a['npix'], a['dp'])[:, a['dc']:a['dc'] + ctx['ch']]
        self._rec('cis_add_slice.' + ctx['form'], 'slice sum', exact(got, ctx['ref']))
        if ctx.get('bad') is not None and not torch.equal(ctx['bad'], ctx['ref']):
            self._control('add_slice.acc_dropped', exact(got, ctx['bad']))

    # ---- flow statistics and the generator input
    def _pre_flow_stats(self, a):
        B, hw = a['B'], a['hw']
        f = self.mem.view(a['flow'], torch.float32, (B, hw, 2)).clone()
        old = self.mem.view(a['stats'], torch.float64, (B, 4)).clone()
        d = f.double()
        ref = old + torch.cat([d.sum(1), (d * d).sum(1)], 1)
        S = old.abs() + torch.cat([d.abs().sum(1), (d * d).sum(1)], 1)
        return dict(ref=ref, S=S, gamma=(hw + 64) * 2.0 ** -53, reads=[f], dests=[(a['stats'], torch.float64, B, 4, 0, 4)])

    def _post_flow_stats(self, a, ctx):
        got = self.mem.view(a['stats'], torch.float64, (a['B'], 4))
        self._rec('cis_flow_stats', 'flow sums', ratio(got, ctx['ref'], ctx['gamma'] * ctx['S']))

    def _pre_pack_generator_input(self, a):
        B, hw = a['B'], a['hw']
        img = self.mem.view(a['image'], torch.float32, (B * hw, 3)).clone()
        f = self.mem.view(a['flow'], torch.float32, (B, hw, 2)).clone()
        d = f.double()
        ref_f = OL.preprocess_flow_batch(d.view(B, hw, 1, 2)).view(B * hw, 2)
        m = d.mean(1, keepdim=True)
        r = 1.0 / ((d - m) ** 2).mean(1, keepdim=True).sqrt()
        S = ((d.abs() + m.abs()) * r).view(B * hw, 2)
        return dict(img=img.to(torch.bfloat16), ref_f=ref_f, S=S, reads=[img, f], dests=[(a['dst'], torch.bfloat16, B * hw, 8, 0, 8)])

    def _post_pack_generator_input(self, a, ctx):
        got = self._bf(a['dst'], a['B'] * a['hw'], 8)
        r = max(exact(got[:, :3], ctx['img']), exact(got[:, 5:], torch.zeros_like(got[:, 5:])))
        r = max(r, ratio(got[:, 3:5], ctx['ref_f'], _bound(ctx['ref_f'], ctx['S'], G_LERP * (1 + 2 ** -7), E_BF16)))
        self._rec('cis_pack_generator_input', 'generator input', r)

    # ---- warp + cost volume
    def _cv_operands(self, a):
        B, h, w, C = a['B'], a['h'], a['w'], a['C']
        Cp = 8 * (-(-C // 8))
        c1 = self.mem.view(a['c1'], torch.bfloat16, (B, h, w, a['c1p']))[..., a['c1o']:a['c1o'] + Cp].clone()
        c2 = self.mem.view(a['c2'], torch.bfloat16, (B, h, w, a['c2p']))[..., a['c2o']:a['c2o'] + Cp].clone()
        flow = self.mem.view(a['flow'], torch.float32, (B, h, w, 2)).clone() if a['flow'] else None
        return c1, c2, flow, Cp

    @staticmethod
    def _cv_pre(c1, wp, C, Cp, R=4):
        x1 = c1.double()
        pre = _corr(x1, wp.W, R) / C
        S = _corr(x1.abs(), wp.W.abs(), R) / C
        bound = (Cp + 6) * U23 * S + _corr(x1.abs(), wp.Werr, R) / C
        return pre, bound

    def _pre_warp_costvol(self, a, R=4):
        C = a['C']
        c1, c2, flow, Cp = self._cv_operands(a)
        wp = _Warp(c2.double(), flow, a['fs'])
        pre, bound = self._cv_pre(c1, wp, C, Cp, R)
        nd = (2 * R + 1) ** 2
        # the window is the (2R+1)^2 channels padded to a multiple of 8: the padding channels must stay exactly 0
        ctx = dict(pre=pre, bound=bound, nd=nd, label='cis_warp_costvol_r' if 'r' in a else 'cis_warp_costvol',
                   reads=[c1, c2] + ([flow] if flow is not None else []),
                   dests=[(a['out'], torch.bfloat16, a['B'] * a['h'] * a['w'], a['op'], a['oo'], a['oo'] + 8 * (-(-nd // 8)))])
        if self.controls is not None and flow is not None and 'warp_costvol.fs_x1.25' not in self.controls:
            ctx['bad'] = self._cv_pre(c1, _Warp(c2.double(), flow, a['fs'], fs_scale=1.25), C, Cp, R)[0]
        if self.controls is not None and R == 1 and 'warp_costvol_r1.dx_outer' not in self.controls:
            # the displacements listed dx outer instead of dy outer
            ctx['dx_outer'] = pre.view(pre.shape[:-1] + (3, 3)).transpose(-1, -2).reshape(pre.shape)
        return ctx

    def _pre_warp_costvol_r(self, a):
        return self._pre_warp_costvol(a, a['r'])

    def _cv_ratio(self, got, pre, bound):
        ref = F.leaky_relu(pre, 0.1)
        amb = pre.abs() <= bound
        err = (got.double() - ref).abs()
        alt = (got.double() - torch.where(pre > 0, 0.1 * pre, pre)).abs()
        err = torch.where(amb, torch.minimum(err, alt), err)
        b = E_BF16 * pre.abs() + bound * (1 + 2 ** -7) + FLOOR
        if not torch.isfinite(got.double()).all():
            return float('inf')
        return float((err / b).max())

    def _post_warp_costvol(self, a, ctx):
        label, nd = ctx['label'], ctx['nd']
        out = self.mem.view(a['out'], torch.bfloat16, (a['B'], a['h'], a['w'], a['op']))
        got = out[..., a['oo']:a['oo'] + nd]
        if not bool((out[..., a['oo'] + nd:a['oo'] + 8 * (-(-nd // 8))].view(torch.int16) == 0).all()):
            self.failures.append('%s launch %d %s: padding channels not +0' % (self.where + (label,)))
        self._rec(label, 'cost volume', self._cv_ratio(got, ctx['pre'], ctx['bound']))
        if 'bad' in ctx:
            self._control('warp_costvol.fs_x1.25', self._cv_ratio(got, ctx['bad'], ctx['bound']))
        if 'dx_outer' in ctx:
            self._control('warp_costvol_r1.dx_outer', self._cv_ratio(got, ctx['dx_outer'], ctx['bound']))
        if self.controls is not None and 'tile.' + label not in self.controls:
            self._control('tile.' + label, self._cv_ratio(_tile(got), ctx['pre'], ctx['bound']))

    def _post_warp_costvol_r(self, a, ctx):
        self._post_warp_costvol(a, ctx)

    def _pre_warp_costvol_bwd(self, a, R=4):
        B, h, w, C = a['B'], a['h'], a['w'], a['C']
        ND = (2 * R + 1) ** 2
        c1, c2, flow, Cp = self._cv_operands(a)
        wp = _Warp(c2.double(), flow, a['fs'])
        pre, bpre = self._cv_pre(c1, wp, C, Cp, R)
        dcorr = self.mem.view(a['dcorr'], torch.bfloat16, (B, h, w, a['dcp']))[..., a['dco']:a['dco'] + ND].clone()
        dc = dcorr.double()
        x1 = c1.double()

        def grads(slope):
            G = dc * slope / C
            amb = 0.9 * dc.abs() / C * (pre.abs() <= bpre)
            dc1 = sum(G[..., k:k + 1] * _shift(wp.W, dy, dx) for k, (dy, dx) in enumerate(_disps(R)))
            dW = sum(_shift(G[..., k:k + 1] * x1, -dy, -dx) for k, (dy, dx) in enumerate(_disps(R)))
            return G, amb, dc1, dW
        G, amb, dc1, dW = grads(torch.where(pre > 0, 1.0, 0.1))
        Wa = wp.W.abs()
        gam = (ND + 6) * U23
        S1 = sum(G[..., k:k + 1].abs() * _shift(Wa, dy, dx) for k, (dy, dx) in enumerate(_disps(R)))
        E1 = sum(amb[..., k:k + 1] * _shift(Wa, dy, dx) + G[..., k:k + 1].abs() * _shift(wp.Werr, dy, dx)
                 for k, (dy, dx) in enumerate(_disps(R)))
        SW = sum(_shift(G[..., k:k + 1].abs() * x1.abs(), -dy, -dx) for k, (dy, dx) in enumerate(_disps(R)))
        EW = sum(_shift(amb[..., k:k + 1] * x1.abs(), -dy, -dx) for k, (dy, dx) in enumerate(_disps(R)))
        errW = gam * SW + EW                               # what the fp32 dwarp may be off by
        npix = B * h * w
        out = dict(reads=[c1, c2, dcorr] + ([flow] if flow is not None else []), dests=[], checks=[],
                   label='cis_warp_costvol_bwd_r' if 'r' in a else 'cis_warp_costvol_bwd')

        def add(p, pitch, off, nch, ref, err, bit, what):
            old = self.mem.view(p, torch.bfloat16, (B, h, w, pitch))[..., off:off + nch].double()
            if a['acc'] & bit:
                ref, err = ref + old, err + gam * old.abs()
            err = err + G_LERP * (ref.abs() + old.abs())
            out['checks'].append((p, pitch, off, nch, ref, err, what))
            out['dests'].append((p, torch.bfloat16, npix, pitch, off, off + nch))
        add(a['dc1'], a['dc1p'], a['dc1o'], C, dc1[..., :C], (gam * S1 + E1)[..., :C], 1, 'dc1')
        if flow is None:
            add(a['dc2'], a['dc2p'], a['dc2o'], C, dW[..., :C], errW[..., :C], 2, 'dc2')
        else:
            dc2 = wp.scatter(dW)
            err2 = wp.scatter(errW) + wp.scatter(dW.abs() * (wp.eps_y + wp.eps_x)[..., None], weights=False) + \
                wp.spread(dW.abs() * wp.amb_pos[..., None])
            add(a['dc2'], a['dc2p'], a['dc2o'], C, dc2[..., :C], err2[..., :C], 2, 'dc2')
            fs = wp.fs
            ay = wp.ay[..., None]
            dy_ = (dW * (wp.bo - wp.t)).sum(-1)
            dx_ = (dW * (ay * (wp.br - wp.bl) + (1 - ay) * (wp.tr - wp.tl))).sum(-1)
            ref = torch.stack([torch.where(wp.pass_y, -fs * dy_, 0.0), torch.where(wp.pass_x, -fs * dx_, 0.0)], -1)
            e = abs(fs) * ((errW * wp.Sc).sum(-1) + (C + 16) * U23 * (dW.abs() * wp.Sc).sum(-1) + (dW.abs() * wp.Werr).sum(-1)
                           + wp.amb_pos * (dW.abs() * 4 * wp.M).sum(-1))
            add(a['dflow'], a['dfp'], a['dfo'], 2, ref, torch.stack([e, e], -1), 4, 'dflow')
            out['dests'] += [(a['ws'], torch.float32, npix, C, 0, C), (a['ds'], torch.float64, npix, C, 0, C)]
        out['dests'].append((a['gs'], torch.float32, npix, ND, 0, ND))
        if self.controls is not None:
            out['bad_dc1'] = grads(torch.ones_like(pre))[2][..., :C] - dc1[..., :C]      # what the ungated gradient adds
        return out

    def _post_warp_costvol_bwd(self, a, ctx):
        B, h, w = a['B'], a['h'], a['w']
        for p, pitch, off, nch, ref, err, what in ctx['checks']:
            got = self.mem.view(p, torch.bfloat16, (B, h, w, pitch))[..., off:off + nch]
            b = E_BF16 * ref.abs() + err * (1 + 2 ** -7)
            self._rec(ctx['label'], what, ratio(got, ref, b))
            if what == 'dc1' and 'bad_dc1' in ctx:
                # the largest over the levels: where the correlations are almost all positive the gate hardly matters
                r = ratio(got, ref + ctx['bad_dc1'], b)
                self.controls['costvol_bwd.gate_one'] = max(r, self.controls.get('costvol_bwd.gate_one', 0.0))

    def _pre_warp_costvol_bwd_r(self, a):
        return self._pre_warp_costvol_bwd(a, a['r'])

    def _post_warp_costvol_bwd_r(self, a, ctx):
        self._post_warp_costvol_bwd(a, ctx)

    # ---- multi-scale flow loss and its backward
    def _ms_levels(self, a, scale=(1.0, 1.0), level_shift=0):
        """Per level i: the fp32 flow read, d = flow - target in fp64 and e = the per-channel bound on the kernel's fp32 d.
        scale / level_shift: corrupted targets (negative controls)."""
        pyr, B, H, W, GH, GW = a['pyr']._obj, a['B'], a['H'], a['W'], a['GH'], a['GW']
        gt = self.mem.view(a['gt'], torch.float32, (B, GH, GW, 2)).clone()
        x = gt.double()
        s = (float(_f32(a['s0'])) * scale[0], float(_f32(a['s1'])) * scale[1])
        out = []
        for i in range(5):
            l = 6 - i
            h, w = H >> l, W >> l
            f = self.mem.view(pyr.flow[i], torch.float32, (B, h, w, 2)).clone()
            (My, Iy), (Mx, Ix) = lerp_axis(GH, h), lerp_axis(GW, w)
            sc = torch.tensor([s[0], s[1]], dtype=torch.float64, device='cuda') * 2.0 ** -(l - level_shift)
            t = apply2(My, Mx, x) * sc
            d = f.double() - t
            e = G_LERP * apply2(Iy, Ix, x.abs()) * sc.abs() + U23 * (f.double().abs() + t.abs())
            out.append(dict(f=f, d=d, e=e, h=h, w=w))
        return gt, out

    @staticmethod
    def _rho(d, e, robust, eps, q):
        """(rho(d), bound on |rho(d') - rho(d)| for |d'_c - d_c| <= e_c) per pixel, fp64."""
        E = e.sum(-1)
        if robust:
            x = d.abs().sum(-1) + eps
            r = x ** q
            return r, q * torch.clamp(x - E, min=eps) ** (q - 1) * E + 2.0 ** -50 * r
        r = torch.sqrt((d * d).sum(-1))
        return r, E + 2.0 ** -50 * r                 # ||.|| is 1-Lipschitz

    def _pre_flow_multiscale_loss(self, a):
        B = a['B']
        robust, eps, q = a['robust'], float(_f32(a['eps'])), float(_f32(a['q']))
        gt, lv = self._ms_levels(a)

        def sums(levels):
            ref, err = [], []
            for L in levels:
                r, er = self._rho(L['d'], L['e'], robust, eps, q)
                hw = L['h'] * L['w']
                ref.append(r.sum((1, 2)))
                err.append(er.sum((1, 2)) + (hw + 128) * 2.0 ** -53 * r.sum((1, 2)))
            return torch.stack(ref, 1), torch.stack(err, 1)
        ref, err = sums(lv)
        ctx = dict(ref=ref, err=err, reads=[gt] + [L['f'] for L in lv],
                   dests=[(a['scratch'], torch.float64, 5 * B, 64, 0, 64), (a['out'], torch.float64, B, 5, 0, 5)])
        if self.controls is not None:
            if float(_f32(a['s0'])) != float(_f32(a['s1'])):
                ctx['bad_axes'] = sums(self._ms_levels(a, scale=(float(_f32(a['s1'])) / float(_f32(a['s0'])),
                                                                float(_f32(a['s0'])) / float(_f32(a['s1']))))[1])[0]
            ctx['bad_level'] = sums(self._ms_levels(a, level_shift=1)[1])[0]
        return ctx

    def _post_flow_multiscale_loss(self, a, ctx):
        got = self.mem.view(a['out'], torch.float64, (a['B'], 5))
        self._rec('cis_flow_multiscale_loss', 'level sums', ratio(got, ctx['ref'], ctx['err']))
        if 'bad_axes' in ctx:
            self._control('ms_loss.axes_swapped', ratio(got, ctx['bad_axes'], ctx['err']))
        if 'bad_level' in ctx:
            self._control('ms_loss.level_scale', ratio(got, ctx['bad_level'], ctx['err']))

    def _ms_grad(self, L, robust, eps, q):
        """(d rho / d flow, its bound, where the kernel's value may be any vector of norm <= 1) per pixel, before the weight."""
        d, e = L['d'], L['e']
        if robust:
            E = e.sum(-1, keepdim=True)
            x = d.abs().sum(-1, keepdim=True) + eps
            Dx = E + U23 * x                                  # the kernel's fp32 |d0| + |d1| + eps
            xl = torch.clamp(x - Dx, min=eps * (1 - U23))
            k = q * x ** (q - 1)
            ek = q * (1 - q) * xl ** (q - 2) * Dx + k * (4 * U23 + 2.0 ** -24 + x.log().abs() * 2.0 ** -24)
            amb = d.abs() <= e                                # sign(d_c) may go either way
            g = torch.where(amb, torch.zeros_like(d), torch.sign(d) * k)
            err = torch.where(amb, q * xl ** (q - 1) * (1 + 2 * U23), ek.expand_as(d))
            return g, err, None
        n = torch.sqrt((d * d).sum(-1, keepdim=True))
        E = e.sum(-1, keepdim=True)
        amb = n <= 4 * E
        g = torch.where(amb, torch.zeros_like(d), d / torch.where(amb, torch.ones_like(n), n))
        err = torch.where(amb, torch.ones_like(d) * (1 + 2.0 ** -20), 2 * E / torch.clamp(n - E, min=FLOOR) + 2.0 ** -21)
        return g, err, amb[..., 0]

    def _pre_flow_multiscale_loss_bwd(self, a, weights=None):
        pyr, B = a['pyr']._obj, a['B']
        robust, eps, q = a['robust'], float(_f32(a['eps'])), float(_f32(a['q']))
        gt, lv = self._ms_levels(a)
        wts = [float(pyr.weight[i]) for i in range(5)]
        checks, dests, reads = [], [], [gt]
        bad = []
        for i, L in enumerate(lv):
            g, err, amb = self._ms_grad(L, robust, eps, q)
            n = B * L['h'] * L['w']
            p, pitch, c0 = pyr.grad[i], pyr.pitch[i], pyr.c_off[i]
            old = self._bf(p, n, pitch)[:, c0:c0 + 2].double().view(B, L['h'], L['w'], 2)
            acc = bool(pyr.accumulate[i])
            ref = wts[i] * g + (old if acc else 0.0)
            e = wts[i] * err * (1 + 2 * U23) + (U23 * (old.abs() + wts[i] * g.abs()) if acc else 0.0)
            checks.append(dict(p=p, pitch=pitch, c0=c0, n=n, shape=(B, L['h'], L['w'], 2), ref=ref, e=e, amb=amb, wt=wts[i], old=old,
                               acc=acc, pads=self.mem.pads(p, pitch, 0, pitch)))
            bad.append(wts[4 - i] * g + (old if acc else 0.0))
            dests.append((p, torch.bfloat16, n, pitch, c0, c0 + 2))
            reads.append(L['f'])
        return dict(checks=checks, dests=dests, reads=reads, bad=bad if wts != wts[::-1] else None)

    def _post_flow_multiscale_loss_bwd(self, a, ctx):
        worst_bad = 0.0
        for i, c in enumerate(ctx['checks']):
            got = self._bf(c['p'], c['n'], c['pitch'])[:, c['c0']:c['c0'] + 2].view(c['shape'])
            b = E_BF16 * c['ref'].abs() + c['e'] * (1 + 2 ** -7)
            self._rec('cis_flow_multiscale_loss_bwd', 'level %d gradient' % (6 - i), ratio(got, c['ref'], b))
            if c['amb'] is not None and bool(c['amb'].any()):
                # where ||d|| is within a few e_d of 0: any vector of norm <= weight
                v = got.double() - (c['old'] if c['acc'] else 0.0)
                nrm = torch.sqrt((v * v).sum(-1))[c['amb']]
                self._rec('cis_flow_multiscale_loss_bwd', 'near-zero norm', float(nrm.max()) / (c['wt'] * (1 + 2 ** -6)))
            if c['pads']:
                pv = self._bf(c['p'], c['n'], c['pitch'])[:, c['pads']]
                if not bool((pv.view(torch.int16) == 0).all()):
                    self.failures.append('%s launch %d cis_flow_multiscale_loss_bwd: level %d gradient padding channels %s not +0'
                                         % (self.where + (6 - i, c['pads'])))
            if ctx['bad'] is not None:
                worst_bad = max(worst_bad, ratio(got, ctx['bad'][i], b))
            self._control('tile.cis_flow_multiscale_loss_bwd', ratio(_tile(got), c['ref'], b))
        if ctx['bad'] is not None:
            self._control('ms_loss_bwd.weights_reversed', worst_bad)

    # ---- TF-Adam with L2 on the kernel segments
    @staticmethod
    def _adam_ref(w, m, v, g0, inseg, decay, lr, b1, b2, eps, t):
        g = g0 + torch.where(inseg, decay * w, torch.zeros_like(w))
        lr_t = lr * (1 - b2 ** t) ** 0.5 / (1 - b1 ** t)
        m1 = b1 * m + (1 - b1) * g
        v1 = b2 * v + (1 - b2) * g * g
        return g, m1, v1, lr_t, w - lr_t * m1 / (v1.sqrt() + eps)

    def _pre_adam_l2(self, a):
        n = a['n']
        snap = [self.mem.view(a[k], torch.float32, (n,)).clone() for k in ('param', 'm', 'v', 'grad')]
        seg = self.mem.view(a['seg'], torch.int64, (a['nseg'], 2)).clone() if a['nseg'] else torch.zeros(0, 2, dtype=torch.int64)
        lr = float(self.mem.view(a['lr'], torch.float32, (1,)))
        step = int(self.mem.view(a['step_state'], torch.int64, (1,)))
        w, m, v, g0 = (x.double() for x in snap)
        inseg = torch.zeros(n, dtype=torch.bool, device='cuda')
        for s0, s1 in seg.tolist():
            inseg[s0:s1] = True
        decay, b1, b2, eps = (float(_f32(a[k])) for k in ('decay', 'beta1', 'beta2', 'eps'))
        t = step + 1
        g, m1, v1, lr_t, w1 = self._adam_ref(w, m, v, g0, inseg, decay, lr, b1, b2, eps, t)
        u = 2.0 ** -24
        e_g = u * (2 * (decay * w).abs() * inseg + g.abs())
        e_m = 2 * u * (b1 * m.abs() + (1 - b1) * g.abs()) + (1 - b1) * e_g
        e_v = 3 * u * (b2 * v + (1 - b2) * g * g) + (1 - b2) * 2 * g.abs() * e_g
        # lr_t: powf within 4 ulp (2^-22 on b^t in [0.5, 1)), 1 - b^t exact (Sterbenz), sqrtf, two products
        rel_lr = 0.5 * 2.0 ** -22 / (1 - b2 ** t) + 2.0 ** -22 / (1 - b1 ** t) + 4 * u
        den = v1.sqrt() + eps
        e_den = torch.minimum(e_v / (2 * v1.sqrt()).clamp(min=FLOOR), e_v.sqrt()) + 2 * u * den
        U = lr_t * m1 / den
        e_U = U.abs() * (rel_lr + 3 * u + e_den / den) + lr_t * e_m / den
        ctx = dict(ref=(w1, m1, v1), err=(u * w1.abs() + e_U, e_m, e_v), grad=snap[3], step=step,
                   reads=snap, dests=[(a[k], torch.float32, 1, n, 0, n) for k in ('param', 'm', 'v')] +
                   [(a['step_state'], torch.int64, 1, 1, 0, 1)])
        if self.controls is not None:
            ctx['bad_decay'] = self._adam_ref(w, m, v, g0, torch.ones_like(inseg), decay, lr, b1, b2, eps, t)[1:]
            if t >= 2:
                ctx['bad_t'] = self._adam_ref(w, m, v, g0, inseg, decay, lr, b1, b2, eps, t - 1)[1:]
        return ctx

    def _post_adam_l2(self, a, ctx):
        n = a['n']
        got = [self.mem.view(a[k], torch.float32, (n,)) for k in ('param', 'm', 'v')]
        for what, x, r, e in zip(('param', 'm', 'v'), got, ctx['ref'], ctx['err']):
            self._rec('cis_adam_l2', what, ratio(x, r, e))
        step = int(self.mem.view(a['step_state'], torch.int64, (1,)))
        self._rec('cis_adam_l2', 'step advanced by one', 0.0 if step == ctx['step'] + 1 else float('inf'))
        self._rec('cis_adam_l2', 'grad unchanged', exact(self.mem.view(a['grad'], torch.float32, (n,)), ctx['grad']))
        for name, key in (('adam.decay_everywhere', 'bad_decay'), ('adam.t_off_by_one', 'bad_t')):
            if key in ctx:
                bad = ctx[key]
                self._control(name, max(ratio(got[0], bad[3], ctx['err'][0]), ratio(got[1], bad[0], ctx['err'][1]),
                                        ratio(got[2], bad[1], ctx['err'][2])))

    # ---- augmentation: parameter rows and the per-pixel pass
    @staticmethod
    def _aug_ranges(r):
        out = {}
        for name, _ in r._fields_:
            v = getattr(r, name)
            out[name] = float(v) if isinstance(v, float) else tuple(float(x) for x in v)
        return out

    def _aug_rows_ratio(self, got, ref):
        """0 / inf for the accepted attempt, the noise key and the zero tail, else max |got - fp32(ref)| / (one fp32 ulp) over
        columns 0..24."""
        import numpy as np
        g = got.cpu().numpy()
        if not (np.array_equal(g[:, 26], ref[:, 26]) and np.array_equal(g[:, 25].view(np.uint32).astype(np.float64), ref[:, 25])
                and not g[:, 27:].any()):
            return float('inf')
        r32 = ref[:, :25].astype(np.float32)
        ulp = np.spacing(np.abs(r32)).astype(np.float64)
        return float((np.abs(g[:, :25].astype(np.float64) - r32.astype(np.float64)) / ulp).max())

    def _pre_flow_aug_params(self, a):
        import flow_aug_ref as AR
        B = a['B']
        t = int(self.mem.view(a['step'], torch.int64, (1,)))
        rg = self._aug_ranges(a['ranges']._obj)
        ref = AR.params(rg, B, a['H'], a['W'], a['sample_offset'], t, a['seed'])
        ctx = dict(ref=ref, t=t, dests=[(a['params'], torch.float32, B, _lib.FLOW_AUG_ROW, 0, _lib.FLOW_AUG_ROW)])
        if self.controls is not None and t >= 1:
            ctx['bad'] = AR.params(rg, B, a['H'], a['W'], a['sample_offset'], 0, a['seed'])
        return ctx

    def _post_flow_aug_params(self, a, ctx):
        got = self.mem.view(a['params'], torch.float32, (a['B'], _lib.FLOW_AUG_ROW))
        self._rec('cis_flow_aug_params', 'parameter rows (fp32 ulps)', self._aug_rows_ratio(got, ctx['ref']))
        if 'bad' in ctx:
            self._control('aug_params.step_frozen', self._aug_rows_ratio(got, ctx['bad']))

    def _pre_flow_augment(self, a):
        import flow_aug_ref as AR
        B, H, W = a['B'], a['H'], a['W']
        src = [self.mem.view(a[k], torch.float32, (B, H, W, c)).clone() for k, c in (('img1', 3), ('img2', 3), ('gt', 2))]
        table = self.mem.view(a['params'], torch.float32, (B, _lib.FLOW_AUG_ROW)).clone()
        P = AR.table_rows(table.cpu().numpy())
        host = [s.cpu().numpy().astype('float64') for s in src]
        ref = AR.augment(*host, P)
        tol = [AR.tolerances(host[0][b], host[1][b], host[2][b], P[b]) for b in range(B)]
        ctx = dict(ref=ref, tol=tol, reads=src + [table], dests=[(a[k], torch.float32, B * H * W, c, 0, c)
                                                                 for k, c in (('img1_out', 3), ('img2_out', 3), ('gt_out', 2))])
        if self.controls is not None:
            # the flow resampled at T1 but not passed through T2^-1: p2 = q + (u, v)
            import numpy as np
            y, x = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing='ij')
            bad = np.empty_like(host[2])
            for b in range(B):
                q1x, q1y = AR.apply(P[b][0:6], x, y)
                gq = AR.bilinear(host[2][b], q1x, q1y)
                bad[b] = np.stack([y - (q1y - gq[..., 0]), x - (q1x - gq[..., 1])], -1)
            ctx['bad'] = bad
        return ctx

    def _post_flow_augment(self, a, ctx):
        import numpy as np
        B, H, W = a['B'], a['H'], a['W']
        got = [self.mem.view(a[k], torch.float32, (B, H, W, c)).cpu().numpy().astype(np.float64)
               for k, c in (('img1_out', 3), ('img2_out', 3), ('gt_out', 2))]
        for f, what in enumerate(('frame 1', 'frame 2', 'flow')):
            r = 0.0
            for b in range(B):
                if not np.isfinite(got[f][b]).all():
                    r = float('inf')
                    break
                r = max(r, float((np.abs(got[f][b] - ctx['ref'][f][b]) / ctx['tol'][b][f]).max()))
            self._rec('cis_flow_augment', what, r)
        if 'bad' in ctx:
            self._control('augment.flow_unmapped', max(float((np.abs(got[2][b] - ctx['bad'][b]) / ctx['tol'][b][2]).max())
                                                       for b in range(B)))

    # ---- unsupervised census + smoothness loss and its backward
    def _unsup_read(self, a):
        B, H, W = a['B'], a['H'], a['W']
        flow = self.mem.view(a['flow'], torch.float32, (2 * B, H, W, 2)).clone()
        i1 = self.mem.view(a['img1'], torch.float32, (B, H, W, 3)).clone()
        i2 = self.mem.view(a['img2'], torch.float32, (B, H, W, 3)).clone()
        return flow, i1, i2

    def _pre_unsup_flow_loss(self, a):
        import unsup_flow_loss_ref as UR
        B, H, W = a['B'], a['H'], a['W']
        N = 2 * B
        flow, i1, i2 = self._unsup_read(a)
        fd = flow.double()
        S, T = UR.directions(i1.double(), i2.double())
        gT = UR.gray(T)
        M, V, lhs, rhs = UR.mask(fd)
        # the occlusion test in fp32: the partner flow h sampled at q (lerps 2^-21 sum |corners|, alpha rounded to fp32), s = f + h
        sp = _unsup_sample(UR.partner(fd), fd)
        h = sp['val']
        eh = 2.0 ** -20 * sp['abs']
        s = fd + h
        e_lhs = (2 * s.abs() * (eh + U23 * s.abs()) + eh * eh).sum(-1) + 3 * U23 * lhs
        e_rhs = (0.01 * (2 * h.abs() * eh + eh * eh)).sum(-1) + abs(float(_f32(0.01)) - 0.01) * ((fd * fd).sum(-1) + (h * h).sum(-1)) \
            + 6 * U23 * rhs
        amb = (lhs - rhs).abs() <= 2 * (e_lhs + e_rhs)
        # T~: lerps of fp32 gray levels (each rounded from double) with fp32 alphas
        st = _unsup_sample(gT.unsqueeze(-1), fd)
        ctx = dict(M=M, V=V, amb=amb, warped=st['val'][..., 0], e_warped=2.0 ** -20 * st['abs'][..., 0], S=S, fd=fd,
                   reads=[flow, i1, i2], dests=[(a[k], torch.float32, N, H * W, 0, H * W) for k in ('warped', 'mask', 'coef')] +
                   [(a['scratch'], torch.float64, N, 128, 0, 128), (a['out'], torch.float64, N, 2, 0, 2)])
        ctx['smooth'] = _unsup_smooth_terms(fd, S)
        return ctx

    def _post_unsup_flow_loss(self, a, ctx):
        import unsup_flow_loss_ref as UR
        B, H, W = a['B'], a['H'], a['W']
        N = 2 * B
        got_w = self.mem.view(a['warped'], torch.float32, (N, H, W))
        got_m = self.mem.view(a['mask'], torch.float32, (N, H, W)).double()
        got_k = self.mem.view(a['coef'], torch.float32, (N, H, W))
        got_s = self.mem.view(a['out'], torch.float64, (N, 2))
        self._rec('cis_unsup_flow_loss', 'warped frame', ratio(got_w, ctx['warped'], ctx['e_warped']))
        # the mask: the fp64 one except where the occlusion test is within its epsilon (the border test is exact: q is formed in
        # double from the fp32 flow on both sides)
        wrong = (got_m != ctx['M']) & ~ctx['amb']
        self._rec('cis_unsup_flow_loss', 'mask', 0.0 if not bool(wrong.any()) and bool(((got_m == 0) | (got_m == 1)).all()) else float('inf'))
        self.unsup_mask = dict(differ=int((got_m != ctx['M']).sum()), near=int(ctx['amb'].sum()), pixels=got_m.numel(),
                               out=int((ctx['V'] == 0).sum()), occluded=int(((ctx['V'] == 1) & (ctx['M'] == 0)).sum()))
        m = torch.where(ctx['amb'], got_m, ctx['M'])
        cen = _census_bound(UR.gray(ctx['S']), got_w.double())
        c, e_c = cen['c'], cen['e']

        def photo(mm):
            # psi = powf(c + 0.01f, 0.4f) and k = 0.4f powf(c + 0.01f, -0.6f): the perturbation Dc of c + 0.01 (the census bound, the
            # fp32 add and the constant 0.01f), the exponents' fp32 constants, powf's 4 ulp and the product's rounding
            Dc = e_c + U23 * (c + 0.01) + abs(float(_f32(0.01)) - 0.01)
            cl = torch.clamp(c - Dc, min=0) + 0.01
            lg = (c + 0.01).log().abs()
            psi = (c + 0.01) ** 0.4
            e_psi = 0.4 * cl ** -0.6 * Dc + psi * (lg * abs(float(_f32(0.4)) - 0.4) + 4 * U23)
            k = 0.4 * (c + 0.01) ** -0.6
            e_k = 0.24 * cl ** -1.6 * Dc + k * (lg * abs(float(_f32(-0.6)) + 0.6) + 4 * U23 + abs(float(_f32(0.4)) - 0.4) / 0.4 + U23)
            return mm * psi, mm * e_psi, mm * k, mm * e_k
        P, eP, K, eK = photo(m)
        self._rec('cis_unsup_flow_loss', 'coef', ratio(got_k, K, eK))
        sm = ctx['smooth']
        hw = H * W
        ref = torch.stack([P.sum((1, 2)), sm['val'].sum((1, 2))], 1)
        err = torch.stack([eP.sum((1, 2)) + (hw + 128) * 2.0 ** -53 * P.sum((1, 2)),
                           sm['err'].sum((1, 2)) + (2 * hw + 128) * 2.0 ** -53 * sm['val'].sum((1, 2))], 1)
        self._rec('cis_unsup_flow_loss', 'direction sums', ratio(got_s, ref, err))
        if self.controls is not None:
            P1, _, K1, _ = photo(torch.ones_like(m))
            bad = torch.stack([P1.sum((1, 2)), sm['val'].sum((1, 2))], 1)
            self._control('unsup.mask_ones', max(ratio(got_s, bad, err), ratio(got_k, K1, eK)))

    def _pre_unsup_flow_loss_bwd(self, a):
        B, H, W = a['B'], a['H'], a['W']
        N = 2 * B
        flow, i1, i2 = self._unsup_read(a)
        warped = self.mem.view(a['warped'], torch.float32, (N, H, W)).clone()
        coef = self.mem.view(a['coef'], torch.float32, (N, H, W)).clone()
        wp, ws = float(_f32(a['w_photo'])), float(_f32(a['w_smooth']))
        r = unsup_bwd_gather(flow.double(), i1.double(), i2.double(), warped.double(), coef.double(), wp, ws, bounds=True)
        return dict(r=r, reads=[flow, i1, i2, warped, coef], dests=[(a['dflow'], torch.float32, N * H * W, 2, 0, 2)])

    def _post_unsup_flow_loss_bwd(self, a, ctx):
        got = self.mem.view(a['dflow'], torch.float32, (2 * a['B'], a['H'], a['W'], 2))
        r = ctx['r']
        self._rec('cis_unsup_flow_loss_bwd', 'dflow', ratio(got, r['ref'], r['err']))
        if self.controls is not None:
            self._control('unsup_bwd.smooth_dropped', ratio(got, r['photo'], r['err']))

    # ---- summary
    def summary(self):
        """{label: dict(count=launches or checks, worst=worst bound ratio)}."""
        return {lab: dict(count=len(rs), worst=max(rs)) for lab, rs in sorted(self.results.items())}


def glue_counts(plan):
    """entry point -> launches of `plan` the glue checker owns."""
    return collections.Counter(op[2] for op in plan.ops if op[2] in ARGS)
