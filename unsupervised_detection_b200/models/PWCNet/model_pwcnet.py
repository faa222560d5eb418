"""Frozen PWC-Net 'lg-6-2' (dense + residual/context) forward on the sm_90a kernels.

Mirrors models/PWCNet/model_pwcnet.py of the reference: extract_features :149-168, warp :173-245 (core_warp.py:153-202),
corr :291-340 (core_costvol.py:20-40), predict_flow :476-506, refine_flow :559-576, deconv :283-286, nn :581-649,
predict_from_img_pairs :61-76.  Forward only: the optimiser var_lists exclude 'pwcnet' (adversarial_learner.py:211-234).

Buffer layout: each pyramid level owns ONE NHWC bf16 buffer that holds the whole DenseNet concat
[act4 32|act3 64|act2 96|act1 128|act0 128|corr 81(+7)|c1 C|up_flow 2,up_feat 2(+4)]; every conv writes its output straight
into its channel slice (tf.concat never materialises), the fused warp+cost-volume kernel writes the 81 correlation
channels, and the 4x4 stride-2 transposed convs of the level above write up_flow/up_feat into the tail.
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
    def __init__(self, store, name='pwcnet'):
        self.name = name
        self.L = {}
        # lvl: pyramid level of the layer's OUTPUT map (selects the experimental narrow n-tiles on the coarse levels, engine.small_bn_cap)
        mk = lambda n, k, ci, co, s=1, d=1, act=ACT_LEAKY, tr=False, lvl=0: self.L.__setitem__(
            n, ConvLayer(store, '%s/%s' % (name, n), k, ci, co, s, d, act, 0.1, tag='', transposed=tr, bn_cap=small_bn_cap(lvl)))
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
        E = {}
        for l in range(FLOW_PRED_LVL, PYR_LVLS + 1):
            E[l] = torch.zeros(N, hs[l][0], hs[l][1], self.level_pitch(l), dtype=torch.bfloat16, device=dev)
        self.level_buf = E
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
                    out = Act(N, hs[l][0], hs[l][1], f, dev, buf=E[l], c_off=C1_OFF, name='c1_%d' % l)
                x = B.conv(self.L['featpyr/conv%db' % l], [x], out=out)
                pyr.append(x)
        B.lane = 0
        P.join()
        self.c1, self.c2 = c1, c2
        B.hold((c1, c2, E))
        up_flow_f32 = None
        self.flows = {}
        for l in range(PYR_LVLS, FLOW_PRED_LVL - 1, -1):
            h, w = hs[l]
            pitch = self.level_pitch(l)
            C = NUM_CHANN[l]
            # ---- warp + cost volume (corr :291-340, warp :173-245)
            scaler = 20.0 / 2 ** l                                              # :616
            P.add('cis_warp_costvol', c1[l].ptr, c1[l].pitch, c1[l].c_off, c2[l].ptr, c2[l].pitch, c2[l].c_off,
                  up_flow_f32.data_ptr() if up_flow_f32 is not None else None, scaler, N, h, w, C, E[l].data_ptr(), pitch, CORR_OFF)
            # ---- DenseNet flow estimator (:476-506)
            for i, co in enumerate(DENSE):
                start = A_TOTAL if i == 0 else A_OFF[i - 1]
                src = Act(N, h, w, 0, dev, buf=E[l], c_off=start, chanmap=self._chanmap(l, start), name='x%d_%d' % (l, i))
                dst = Act(N, h, w, co, dev, buf=E[l], c_off=A_OFF[i], name='act%d_%d' % (l, i))
                B.conv(self.L['predict_flow/conv%d_%d' % (l, i)], [src], out=dst)
            upfeat = Act(N, h, w, 0, dev, buf=E[l], c_off=0, chanmap=self._chanmap(l, 0), name='upfeat%d' % l)
            flow_raw = B.f32(N, h, w, 2)
            B.conv(self.L['predict_flow/flow%d' % l], [upfeat], outf=flow_raw, want_bf16=False)
            # ---- context network (:559-576): flow += ctx(upfeat)
            x = upfeat
            for i in range(1, 7):
                x = B.conv(self.L['ctxt/dc_conv%d%d' % (l, i)], [x])
            flow = B.f32(N, h, w, 2)
            flow_bf = B.conv(self.L['ctxt/dc_conv%d7' % l], [x], addf=flow_raw, outf=flow)
            self.flows[l] = flow
            if l != FLOW_PRED_LVL:
                # ---- 4x4 stride-2 transposed convs into the next level's buffer tail (:634-635)
                nh, nw = hs[l - 1]
                tail = C1_OFF + NUM_CHANN[l - 1]
                up_flow_f32 = B.f32(N, nh, nw, 2)
                o1 = Act(N, nh, nw, 2, dev, buf=E[l - 1], c_off=tail, chanmap=[0, 1], name='up_flow%d' % l)
                o2 = Act(N, nh, nw, 2, dev, buf=E[l - 1], c_off=tail + 2, chanmap=[0, 1], name='up_feat%d' % l)
                assert (nh, nw) == (2 * h, 2 * w), 'PWC-Net needs H, W divisible by 64'
                B.conv_transpose(self.L['upsample/up_flow%d' % l], flow_bf, out=o1, outf=up_flow_f32)
                B.conv_transpose(self.L['upsample/up_feat%d' % l], upfeat, out=o2)
            else:
                s = 2 ** FLOW_PRED_LVL
                assert (h * s, w * s) == (H, W)
                P.add('cis_resize_bilinear_f32', flow.data_ptr(), N, h, w, 2, flow_out.data_ptr(), H, W, float(s))   # :646
        return flow_out
