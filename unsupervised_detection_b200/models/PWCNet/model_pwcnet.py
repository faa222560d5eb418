"""PWC-Net (reference options: dense connections, residual/context network, search range) on the sm_90a kernels.

Mirrors models/PWCNet/model_pwcnet.py of the reference: extract_features :149-168, warp :173-245 (core_warp.py:153-202),
corr :291-340 (core_costvol.py:20-40), predict_flow :476-506, refine_flow :559-576, deconv :283-286, nn :581-649,
predict_from_img_pairs :61-76.  `ModelPWCNet(name, options)` is the reference's public class; `PWCNetBuilder` emits the launch lists for
one option set into a Builder (the step graph and the function-level runner use it).  The training step keeps PWC-Net frozen, as the
reference does (its optimiser var_lists exclude 'pwcnet', adversarial_learner.py:211-234): the step graph builds
PWCNetBuilder(trainable=False), forward only.  trainable=True tags every layer 'P' and records the backward on the builder's tape (the
function-level predict_from_img_pairs, models/functional.py): gradients reach every pwcnet/* parameter and both images.

Options (the reference's _DEFAULT_PWCNET_TEST_OPTIONS keys, :8-19): use_dense_cx, use_res_cx and search_range 1..4 are supported, in all
combinations; pyr_lvls = 6 and flow_pred_lvl = 2 are the only pyramid values (every published checkpoint uses them).
  * use_dense_cx=False: conv{l}_i (i >= 1) reads act_{i-1} alone, and flow{l}, ctxt/dc_conv{l}1 and up_feat{l} read act4 (upfeat = act, :502).
  * use_res_cx=False: levels above flow_pred_lvl have no context network (nn :606-642); predict_flow/flow{l} writes the level's fp32 flow and
    the bf16 flow up_flow{l} reads.  The prediction level keeps its context network (refine_flow is unconditional there, :636-639).
  * search_range r: the correlation has (2r+1)^2 channels, dy outer.

Buffer layout: each pyramid level owns ONE NHWC bf16 buffer that holds the whole DenseNet concat
[act4 32|act3 64|act2 96|act1 128|act0 128|corr (2r+1)^2 (padded to 8)|c1 C|up_flow 2,up_feat 2(+4)] for every option set; every conv
writes its output straight into its channel slice (tf.concat never materialises), the fused warp+cost-volume kernel writes the correlation
channels, and the 4x4 stride-2 transposed convs of the level above write up_flow/up_feat into the tail.  Without dense connections only
the source views change.

Backward (trainable): level buffer E[l] has a gradient buffer dE[l] of the same layout, zeroed once per backward.  Every view of E[l] has
the same slice of dE[l] as its gradient and counts as written from the start, so every data gradient into it accumulates; in reverse tape
order all consumers of an activation run before its producer's backward.  With a context network, the two fp32 flow heads
(predict_flow/flow{l} and the dc_conv{l}7 residual, flow = dc7(x) + flow_raw) both take the gradient of the level's bf16 flow as their
output gradient; without one, predict_flow/flow{l} owns that bf16 flow and its gradient.
"""
import collections

import torch

from ...engine import ConvLayer, Act, ACT_NONE, ACT_LEAKY, small_bn_cap

NUM_CHANN = [None, 16, 32, 64, 96, 128, 196]       # model_pwcnet.py:151
PYR_LVLS, FLOW_PRED_LVL, SEARCH_RANGE = 6, 2, 4    # _DEFAULT_PWCNET_TEST_OPTIONS :8-19 (the only pyramid values supported)
DENSE = (128, 128, 96, 64, 32)                     # predict_flow conv widths :484-502
CTX = ((128, 1), (128, 2), (128, 4), (96, 8), (64, 16), (32, 1), (2, 1))   # refine_flow :562-574
A_OFF = (320, 192, 96, 32, 0)                      # channel offset of dense activation i inside the level buffer
A_TOTAL = 448
CORR_OFF, CORR_PAD = 448, 88                       # CORR_PAD, C1_OFF: the default search range 4 (PWCNetBuilder.corr_pad / c1_off)
C1_OFF = CORR_OFF + CORR_PAD

# The reference's module default (model_pwcnet.py:8-19).  ModelPWCNet() and the training / inference graphs read it, so a network is
# selected the reference's way, by setting these values.  verbose and ckpt_path are accepted and ignored (weights come from --flow_ckpt).
_DEFAULT_PWCNET_TEST_OPTIONS = {
    'verbose': False,
    'ckpt_path': './models/PWCNet/checkpoint/pwcnet-sm-6-2-cyclic-chairsthingsmix/pwcnet.ckpt-49000',
    'pyr_lvls': 6,
    'flow_pred_lvl': 2,
    'search_range': 4,
    'use_dense_cx': True,
    'use_res_cx': True,
}

PWCOptions = collections.namedtuple('PWCOptions', 'pyr_lvls flow_pred_lvl search_range use_dense_cx use_res_cx')
_LG = PWCOptions(PYR_LVLS, FLOW_PRED_LVL, SEARCH_RANGE, True, True)     # values of keys an options dict leaves out


def normalize_options(options=None):
    """Options dict (the reference's keys; None = the current _DEFAULT_PWCNET_TEST_OPTIONS) -> PWCOptions, the hashable form every plan
    and runner key uses.  Keys outside PWCOptions are ignored; values outside the supported set raise ValueError."""
    if isinstance(options, PWCOptions):
        return options
    o = _DEFAULT_PWCNET_TEST_OPTIONS if options is None else options
    get = lambda k: o.get(k, getattr(_LG, k))
    if get('pyr_lvls') != PYR_LVLS or get('flow_pred_lvl') != FLOW_PRED_LVL:
        raise ValueError('PWC-Net: pyr_lvls=%r, flow_pred_lvl=%r not supported; supported: pyr_lvls=%d, flow_pred_lvl=%d'
                         % (get('pyr_lvls'), get('flow_pred_lvl'), PYR_LVLS, FLOW_PRED_LVL))
    r = get('search_range')
    if isinstance(r, bool) or r not in (1, 2, 3, 4):
        raise ValueError('PWC-Net: search_range=%r not supported; supported: 1, 2, 3, 4' % (r,))
    return PWCOptions(PYR_LVLS, FLOW_PRED_LVL, int(r), bool(get('use_dense_cx')), bool(get('use_res_cx')))


class _PredictFromImgPairs(object):
    """ModelPWCNet.predict_from_img_pairs in both call forms: on an instance it runs that instance's options (the reference's
    `ModelPWCNet().predict_from_img_pairs(img1s, img2s)`), unbound on the class it runs the default options."""

    def __get__(self, obj, cls):
        from .. import functional

        def predict_from_img_pairs(img_1, img_2, params=None, name=None):
            """model_pwcnet.py:39-76 of the reference: flow img_1 -> img_2 for batches of NHWC images in [-0.5, 0.5] (function-level
            API, see models/functional.py; the training step uses PWCNetBuilder inside its static graph instead)."""
            if obj is None:
                return functional.predict_from_img_pairs(img_1, img_2, name or 'pwcnet', params)
            return functional.predict_from_img_pairs(img_1, img_2, name or obj.name, params, options=obj.options)
        return predict_from_img_pairs


class ModelPWCNet(object):
    """The reference's public class: ModelPWCNet(name='pwcnet', options=_DEFAULT_PWCNET_TEST_OPTIONS).  The options are checked here
    (ValueError outside the supported set) and `predict_from_img_pairs` runs them."""

    def __init__(self, name='pwcnet', options=_DEFAULT_PWCNET_TEST_OPTIONS):
        if not isinstance(name, str):
            raise TypeError('ModelPWCNet(name, options) takes the reference\'s arguments; the launch-list builder is PWCNetBuilder(store, ...)')
        self.name = name
        self.opts = options
        self.options = normalize_options(options)

    predict_from_img_pairs = _PredictFromImgPairs()


class PWCNetBuilder(object):
    """Layers and launch lists of one PWC-Net option set (options: a dict with the reference's keys, a PWCOptions, or None = the current
    _DEFAULT_PWCNET_TEST_OPTIONS).  Layout values that depend on the options are attributes: corr_pad, c1_off, level_pitch(l)."""

    def __init__(self, store, name='pwcnet', trainable=False, options=None):
        self.name = name
        self.trainable = trainable
        self.options = o = normalize_options(options)
        self.search_range = r = o.search_range
        self.ndisp = (2 * r + 1) ** 2                     # correlation channels
        self.corr_pad = -(-self.ndisp // 8) * 8           # their slice of the level buffer
        self.c1_off = CORR_OFF + self.corr_pad
        self.L = {}
        tag = 'P' if trainable else ''
        # lvl: pyramid level of the layer's OUTPUT map (selects the experimental narrow n-tiles on the coarse levels, engine.small_bn_cap)
        mk = lambda n, k, ci, co, s=1, d=1, act=ACT_LEAKY, tr=False, lvl=0: self.L.__setitem__(
            n, ConvLayer(store, '%s/%s' % (name, n), k, ci, co, s, d, act, 0.1, tag=tag, transposed=tr, bn_cap=small_bn_cap(lvl)))
        cin = 3
        for l in range(1, PYR_LVLS + 1):
            f = NUM_CHANN[l]
            mk('featpyr/conv%da' % l, 3, cin, f, 2, lvl=l)
            mk('featpyr/conv%daa' % l, 3, f, f, lvl=l)
            mk('featpyr/conv%db' % l, 3, f, f, lvl=l)
            cin = f
        for l in range(PYR_LVLS, FLOW_PRED_LVL - 1, -1):
            c = self.ndisp if l == PYR_LVLS else self.ndisp + NUM_CHANN[l] + 4
            for i, co in enumerate(DENSE):
                mk('predict_flow/conv%d_%d' % (l, i), 3, c, co, lvl=l)
                c = c + co if o.use_dense_cx else co      # c: width of upfeat after the last conv
            mk('predict_flow/flow%d' % l, 3, c, 2, act=ACT_NONE)
            if self.has_context(l):
                cc = c
                for i, (co, d) in enumerate(CTX, start=1):
                    mk('ctxt/dc_conv%d%d' % (l, i), 3, cc, co, 1, d, ACT_NONE if i == 7 else ACT_LEAKY, lvl=l)
                    cc = co
            if l != FLOW_PRED_LVL:
                mk('upsample/up_flow%d' % l, 4, 2, 2, act=ACT_NONE, tr=True)
                mk('upsample/up_feat%d' % l, 4, c, 2, act=ACT_NONE, tr=True)

    def all_layers(self):
        return list(self.L.values())

    def has_context(self, l):
        """refine_flow runs at every level with use_res_cx, and always at the prediction level (nn :606-642)."""
        return self.options.use_res_cx or l == FLOW_PRED_LVL

    def level_pitch(self, l):
        return A_TOTAL + self.corr_pad + (0 if l == PYR_LVLS else NUM_CHANN[l] + 8)

    def _chanmap(self, l, start):
        """Packed position -> original channel of the DenseNet concat seen from channel `start` of the level buffer."""
        n_a = A_TOTAL - start
        nd = self.ndisp
        cm = list(range(n_a)) + [n_a + j for j in range(nd)] + [-1] * (self.corr_pad - nd)
        if l != PYR_LVLS:
            C = NUM_CHANN[l]
            cm += [n_a + nd + j for j in range(C)] + [n_a + nd + C + j for j in range(4)] + [-1] * 4
        return cm

    def _costvol_op(self, name):
        """The warp + cost-volume entry point and its trailing arguments: the range-free R = 4 one for the default range."""
        return (name, ()) if self.search_range == SEARCH_RANGE else (name + '_r', (self.search_range,))

    def build(self, B, img1_8, img2_8, flow_out):
        """img*_8: Act [N,H,W,8] = image + 0.5 (adapt_x :39-56); flow_out: fp32 [N,H,W,2] <- flow_pred (nn :642-647)."""
        dev = B.device
        N, H, W = img1_8.N, img1_8.H, img1_8.W
        P = B.fwd
        hs = [None] + [(-(-H // 2 ** l), -(-W // 2 ** l)) for l in range(1, PYR_LVLS + 1)]
        E, dE, written = {}, {}, {}
        for l in range(FLOW_PRED_LVL, PYR_LVLS + 1):
            E[l] = torch.zeros(N, hs[l][0], hs[l][1], self.level_pitch(l), dtype=torch.bfloat16, device=dev)
            if self.trainable:
                dE[l] = torch.zeros_like(E[l])
                written[l] = {'P': True}          # shared by every view of E[l]: dE[l] is zeroed, every gradient into it accumulates
        self.level_buf, self.level_grad = E, dE

        def view(l, C, c_off, chanmap=None, name=''):
            a = Act(N, hs[l][0], hs[l][1], C, dev, buf=E[l], c_off=c_off, chanmap=chanmap, name=name)
            if self.trainable:      # written by tagged layers / the cost volume: their gradients flow back through every view
                a.dep, a.grad_buf, a.grad_written = frozenset({'P'}), dE[l], written[l]
            return a
        # ---- feature pyramids (shared weights; frame 1 features land inside the level buffers)
        c1, c2 = [None], [None]
        for pyr, x, first in ((c1, img1_8, True), (c2, img2_8, False)):
            B.lane = 0 if first else 1       # the two pyramids are independent: frame 2 runs on the side stream
            for l in range(1, PYR_LVLS + 1):
                f = NUM_CHANN[l]
                x = B.conv(self.L['featpyr/conv%da' % l], [x])
                x = B.conv(self.L['featpyr/conv%daa' % l], [x])
                out = None
                if first and FLOW_PRED_LVL <= l < PYR_LVLS:
                    out = view(l, f, self.c1_off, name='c1_%d' % l)
                x = B.conv(self.L['featpyr/conv%db' % l], [x], out=out)
                pyr.append(x)
        B.lane = 0
        P.join()
        self.c1, self.c2 = c1, c2
        B.hold((c1, c2, E))
        up_flow_f32 = up_flow = None
        self.flows, self.flows_bf = {}, {}
        for l in range(PYR_LVLS, FLOW_PRED_LVL - 1, -1):
            h, w = hs[l]
            pitch = self.level_pitch(l)
            C = NUM_CHANN[l]
            # ---- warp + cost volume (corr :291-340, warp :173-245)
            scaler = 20.0 / 2 ** l                                              # :616
            op, rng = self._costvol_op('cis_warp_costvol')
            P.add(op, c1[l].ptr, c1[l].pitch, c1[l].c_off, c2[l].ptr, c2[l].pitch, c2[l].c_off,
                  up_flow_f32.data_ptr() if up_flow_f32 is not None else None, scaler, N, h, w, C, E[l].data_ptr(), pitch, CORR_OFF, *rng)
            if self.trainable:
                B.tape.append(lambda bp, m, l=l, fl=up_flow_f32, uf=up_flow, s_=scaler: self._costvol_bwd(bp, m, l, fl, uf, s_))
            # ---- flow estimator (:476-506): with dense connections each conv reads the whole concat behind its output slice, without them
            # conv{l}_0 reads [corr | c1 | up_flow, up_feat] and conv{l}_i the previous activation alone
            dense = self.options.use_dense_cx
            for i, co in enumerate(DENSE):
                if i == 0 or dense:
                    start = A_TOTAL if i == 0 else A_OFF[i - 1]
                    src = view(l, 0, start, chanmap=self._chanmap(l, start), name='x%d_%d' % (l, i))
                else:
                    src = view(l, DENSE[i - 1], A_OFF[i - 1], name='x%d_%d' % (l, i))
                dst = view(l, co, A_OFF[i], name='act%d_%d' % (l, i))
                B.conv(self.L['predict_flow/conv%d_%d' % (l, i)], [src], out=dst)
            if dense:
                upfeat = view(l, 0, 0, chanmap=self._chanmap(l, 0), name='upfeat%d' % l)
            else:
                upfeat = view(l, DENSE[-1], A_OFF[-1], name='upfeat%d' % l)      # upfeat = act (:502)
            if self.has_context(l):
                flow_raw = B.f32(N, h, w, 2)
                # bf16 copy of the refined flow (input of up_flow); its gradient is also the gradient of flow_raw
                flow_bf = B.new_act(N, h, w, 2, name='ctxt/dc_conv%d7' % l)
                B.conv(self.L['predict_flow/flow%d' % l], [upfeat], outf=flow_raw, want_bf16=False, grad_out=flow_bf)
                # ---- context network (:559-576): flow += ctx(upfeat)
                x = upfeat
                for i in range(1, 7):
                    x = B.conv(self.L['ctxt/dc_conv%d%d' % (l, i)], [x])
                flow = B.f32(N, h, w, 2)
                B.conv(self.L['ctxt/dc_conv%d7' % l], [x], addf=flow_raw, outf=flow, out=flow_bf)
            else:
                # no context network: the flow head writes the level's fp32 flow and the bf16 flow up_flow reads, and owns its gradient
                flow = B.f32(N, h, w, 2)
                flow_bf = B.new_act(N, h, w, 2, name='predict_flow/flow%d' % l)
                B.conv(self.L['predict_flow/flow%d' % l], [upfeat], outf=flow, out=flow_bf)
            self.flows[l], self.flows_bf[l] = flow, flow_bf
            if l != FLOW_PRED_LVL:
                # ---- 4x4 stride-2 transposed convs into the next level's buffer tail (:634-635)
                nh, nw = hs[l - 1]
                tail = self.c1_off + NUM_CHANN[l - 1]
                up_flow_f32 = B.f32(N, nh, nw, 2)
                o1 = view(l - 1, 2, tail, chanmap=[0, 1], name='up_flow%d' % l)
                o2 = view(l - 1, 2, tail + 2, chanmap=[0, 1], name='up_feat%d' % l)
                up_flow = o1
                assert (nh, nw) == (2 * h, 2 * w), 'PWC-Net needs H, W divisible by 64'
                B.conv_transpose(self.L['upsample/up_flow%d' % l], flow_bf, out=o1, outf=up_flow_f32)
                B.conv_transpose(self.L['upsample/up_feat%d' % l], upfeat, out=o2)
            else:
                s = 2 ** FLOW_PRED_LVL
                assert (h * s, w * s) == (H, W)
                P.add('cis_resize_bilinear_f32', flow.data_ptr(), N, h, w, 2, flow_out.data_ptr(), H, W, float(s))   # :646
        if self.trainable:
            # scratch of the warp + cost-volume backward (levels run one after another on one stream): gated correlation gradient,
            # gradient of the warped features, fp64 scatter sums
            npix = max(N * hs[l][0] * hs[l][1] for l in range(FLOW_PRED_LVL, PYR_LVLS + 1))
            npc = max(N * hs[l][0] * hs[l][1] * NUM_CHANN[l] for l in range(FLOW_PRED_LVL, PYR_LVLS))
            self.cv_scratch = (B.f32(npix * self.ndisp), B.f32(npc), B.hold(torch.zeros(npc, dtype=torch.float64, device=dev)))
        return flow_out

    def _costvol_bwd(self, bp, mode, l, up_flow_f32, up_flow, scaler):
        """Transpose of the level-l warp + cost volume: dc1 and dc2 into the pyramid gradients, d(up_flow) into the up_flow gradient slice
        of dE[l] (its second consumer after the DenseNet convs), the correlation gradient read from the corr slice of dE[l]."""
        if mode != 'P':
            return
        c1, c2, N = self.c1[l], self.c2[l], self.c1[l].N
        h, w = c1.H, c1.W
        g1, g2 = c1.get_grad(), c2.get_grad()
        acc = (1 if c1.grad_written.get(mode) else 0) | (2 if c2.grad_written.get(mode) else 0)
        gf = (None, 0, 0)
        if up_flow_f32 is not None:
            g = up_flow.get_grad()
            gf = (g.ptr, g.pitch, g.c_off)
            acc |= 4 if up_flow.grad_written.get(mode) else 0
        gs, ws, ds = self.cv_scratch
        op, rng = self._costvol_op('cis_warp_costvol_bwd')
        bp.add(op, c1.ptr, c1.pitch, c1.c_off, c2.ptr, c2.pitch, c2.c_off,
               up_flow_f32.data_ptr() if up_flow_f32 is not None else None, scaler, N, h, w, NUM_CHANN[l],
               self.level_grad[l].data_ptr(), self.level_pitch(l), CORR_OFF, g1.ptr, g1.pitch, g1.c_off, g2.ptr, g2.pitch, g2.c_off,
               gf[0], gf[1], gf[2], acc, gs.data_ptr(), ws.data_ptr() if up_flow_f32 is not None else None,
               ds.data_ptr() if up_flow_f32 is not None else None, *rng)
        c1.grad_written[mode] = c2.grad_written[mode] = True
