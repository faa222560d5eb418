"""PWC-Net 'lg-6-2' (dense + residual/context) on the sm_90a kernels.

Mirrors models/PWCNet/model_pwcnet.py of the reference: extract_features :149-168, warp :173-245 (core_warp.py:153-202),
corr :291-340 (core_costvol.py:20-40), predict_flow :476-506, refine_flow :559-576, deconv :283-286, nn :581-649,
predict_from_img_pairs :61-76.  The training step keeps PWC-Net frozen, as the reference does (its optimiser var_lists exclude 'pwcnet',
adversarial_learner.py:211-234): the step graph builds ModelPWCNet(trainable=False), forward only.  trainable=True tags every layer 'P'
and records the backward on the builder's tape (the function-level predict_from_img_pairs, models/functional.py): gradients reach
every pwcnet/* parameter and both images.

Buffer layout: each pyramid level owns ONE NHWC bf16 buffer that holds the whole DenseNet concat
[act4 32|act3 64|act2 96|act1 128|act0 128|corr 81(+7)|c1 C|up_flow 2,up_feat 2(+4)]; every conv writes its output straight
into its channel slice (tf.concat never materialises), the fused warp+cost-volume kernel writes the 81 correlation
channels, and the 4x4 stride-2 transposed convs of the level above write up_flow/up_feat into the tail.

Backward (trainable): level buffer E[l] has a gradient buffer dE[l] of the same layout, zeroed once per backward.  Every view of E[l] has
the same slice of dE[l] as its gradient and counts as written from the start, so every data gradient into it accumulates; in reverse tape
order all consumers of an activation run before its producer's backward.  The two fp32 flow heads (predict_flow/flow{l} and the
dc_conv{l}7 residual, flow = dc7(x) + flow_raw) both take the gradient of the level's bf16 flow as their output gradient.
"""
import torch

from ...engine import ConvLayer, Act, ACT_NONE, ACT_LEAKY, small_bn_cap

NUM_CHANN = [None, 16, 32, 64, 96, 128, 196]       # model_pwcnet.py:151
PYR_LVLS, FLOW_PRED_LVL, SEARCH_RANGE = 6, 2, 4    # _DEFAULT_PWCNET_TEST_OPTIONS :8-19
DENSE = (128, 128, 96, 64, 32)                     # predict_flow conv widths :484-502
CTX = ((128, 1), (128, 2), (128, 4), (96, 8), (64, 16), (32, 1), (2, 1))   # refine_flow :562-574
A_OFF = (320, 192, 96, 32, 0)                      # channel offset of dense activation i inside the level buffer
A_TOTAL = 448
CORR_OFF, CORR_PAD = 448, 88
C1_OFF = CORR_OFF + CORR_PAD


class ModelPWCNet(object):
    def __init__(self, store, name='pwcnet', trainable=False):
        self.name = name
        self.trainable = trainable
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
            c = 81 if l == PYR_LVLS else 81 + NUM_CHANN[l] + 4
            for i, co in enumerate(DENSE):
                mk('predict_flow/conv%d_%d' % (l, i), 3, c, co, lvl=l)
                c += co
            mk('predict_flow/flow%d' % l, 3, c, 2, act=ACT_NONE)
            cc = c
            for i, (co, d) in enumerate(CTX, start=1):
                mk('ctxt/dc_conv%d%d' % (l, i), 3, cc, co, 1, d, ACT_NONE if i == 7 else ACT_LEAKY, lvl=l)
                cc = co
            if l != FLOW_PRED_LVL:
                mk('upsample/up_flow%d' % l, 4, 2, 2, act=ACT_NONE, tr=True)
                mk('upsample/up_feat%d' % l, 4, c, 2, act=ACT_NONE, tr=True)

    def all_layers(self):
        return list(self.L.values())

    @staticmethod
    def predict_from_img_pairs(img_1, img_2, params=None, name='pwcnet'):
        """model_pwcnet.py:39-76 of the reference: flow img_1 -> img_2 for batches of NHWC images in [-0.5, 0.5] (function-level API,
        see models/functional.py; the training step uses the `build` method below inside its static graph instead)."""
        from .. import functional
        return functional.predict_from_img_pairs(img_1, img_2, name, params)

    @staticmethod
    def level_pitch(l):
        return A_TOTAL + CORR_PAD + (0 if l == PYR_LVLS else NUM_CHANN[l] + 8)

    @staticmethod
    def _chanmap(l, start):
        """Packed position -> original channel of the DenseNet concat seen from channel `start` of the level buffer."""
        n_a = A_TOTAL - start
        cm = list(range(n_a)) + [n_a + j for j in range(81)] + [-1] * 7
        if l != PYR_LVLS:
            C = NUM_CHANN[l]
            cm += [n_a + 81 + j for j in range(C)] + [n_a + 81 + C + j for j in range(4)] + [-1] * 4
        return cm

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
                    out = view(l, f, C1_OFF, name='c1_%d' % l)
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
            P.add('cis_warp_costvol', c1[l].ptr, c1[l].pitch, c1[l].c_off, c2[l].ptr, c2[l].pitch, c2[l].c_off,
                  up_flow_f32.data_ptr() if up_flow_f32 is not None else None, scaler, N, h, w, C, E[l].data_ptr(), pitch, CORR_OFF)
            if self.trainable:
                B.tape.append(lambda bp, m, l=l, fl=up_flow_f32, uf=up_flow, s_=scaler: self._costvol_bwd(bp, m, l, fl, uf, s_))
            # ---- DenseNet flow estimator (:476-506)
            for i, co in enumerate(DENSE):
                start = A_TOTAL if i == 0 else A_OFF[i - 1]
                src = view(l, 0, start, chanmap=self._chanmap(l, start), name='x%d_%d' % (l, i))
                dst = view(l, co, A_OFF[i], name='act%d_%d' % (l, i))
                B.conv(self.L['predict_flow/conv%d_%d' % (l, i)], [src], out=dst)
            upfeat = view(l, 0, 0, chanmap=self._chanmap(l, 0), name='upfeat%d' % l)
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
            self.flows[l], self.flows_bf[l] = flow, flow_bf
            if l != FLOW_PRED_LVL:
                # ---- 4x4 stride-2 transposed convs into the next level's buffer tail (:634-635)
                nh, nw = hs[l - 1]
                tail = C1_OFF + NUM_CHANN[l - 1]
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
            self.cv_scratch = (B.f32(npix * 81), B.f32(npc), B.hold(torch.zeros(npc, dtype=torch.float64, device=dev)))
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
        bp.add('cis_warp_costvol_bwd', c1.ptr, c1.pitch, c1.c_off, c2.ptr, c2.pitch, c2.c_off,
               up_flow_f32.data_ptr() if up_flow_f32 is not None else None, scaler, N, h, w, NUM_CHANN[l],
               self.level_grad[l].data_ptr(), self.level_pitch(l), CORR_OFF, g1.ptr, g1.pitch, g1.c_off, g2.ptr, g2.pitch, g2.c_off,
               gf[0], gf[1], gf[2], acc, gs.data_ptr(), ws.data_ptr() if up_flow_f32 is not None else None,
               ds.data_ptr() if up_flow_f32 is not None else None)
        c1.grad_written[mode] = c2.grad_written[mode] = True
