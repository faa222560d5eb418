"""Generator (mask) and recover (flow-inpainter) networks on the sm_90a conv engine.

Mirrors models/nets.py of the reference (generator_net :4-42, recover_net :45-110) and the layer primitives of
models/utils/convolution_utils.py (gen_conv :26-53, gen_deconv :55-75, conv :77-85, deconv :87-90); same layer names,
shapes and concat orders.  Activations are bf16 NHWC in HBM, every layer is one cis_conv_igemm launch with
bias / BN-affine / ELU / leaky / skip-add fused into the epilogue.
"""
from ..engine import ConvLayer, ACT_NONE, ACT_ELU, ACT_LEAKY

# name, cin, cout, ksize, stride, rate   (nets.py:19-36)
GEN_LAYERS = [
    ('conv1', 5, 32, 5, 1, 1), ('conv2_downsample', 32, 64, 3, 2, 1), ('conv3', 64, 64, 3, 1, 1),
    ('conv4_downsample', 64, 128, 3, 2, 1), ('conv5', 128, 128, 3, 1, 1), ('conv6', 128, 128, 3, 1, 1),
    ('conv7_atrous', 128, 128, 3, 1, 2), ('conv8_atrous', 128, 128, 3, 1, 4), ('conv9_atrous', 128, 128, 3, 1, 8),
    ('conv10_atrous', 128, 128, 3, 1, 16), ('conv11', 128, 128, 3, 1, 1), ('conv12', 128, 128, 3, 1, 1),
    ('conv13_upsample', 128, 64, 3, 1, 1), ('conv14', 64, 64, 3, 1, 1), ('conv15_upsample', 64, 32, 3, 1, 1),
    ('conv16', 32, 16, 3, 1, 1), ('conv17', 16, 2, 3, 1, 1)]


class GeneratorNet(object):
    """generator_net (nets.py:4-42).  gen_conv = conv2d SAME + BN(inference: y = gamma*x/sqrt(1+1e-3)+beta, folded into the
    weights) + ELU; conv17 has identity activation and feeds softmax(x/10)[...,0] == sigmoid((x0-x1)/10)."""

    def __init__(self, store, scope='MaskNet'):
        self.scope = scope
        self.layers = {}
        for name, cin, cout, k, s, r in GEN_LAYERS:
            act = ACT_NONE if name == 'conv17' else ACT_ELU
            self.layers[name] = ConvLayer(store, '%s/%s' % (scope, name), k, cin, cout, s, r, act, tag='G', bn=True)

    def all_layers(self):
        return list(self.layers.values())

    def build(self, B, x_in, mask_out):
        """x_in: Act [N,H,W,8] = concat(image 3, normalised flow 2); mask_out: fp32 [N,H,W,1] device tensor."""
        L = self.layers
        x_0 = B.conv(L['conv1'], [x_in])
        x = B.conv(L['conv2_downsample'], [x_0])
        x_1 = B.conv(L['conv3'], [x])
        x = B.conv(L['conv4_downsample'], [x_1])
        x = B.conv(L['conv5'], [x])
        x_2 = B.conv(L['conv6'], [x])
        x = B.conv(L['conv7_atrous'], [x_2])
        x = B.conv(L['conv8_atrous'], [x])
        x = B.conv(L['conv9_atrous'], [x])
        x = B.conv(L['conv10_atrous'], [x])
        x = B.conv(L['conv11'], [x], post_add=x_2)          # nets.py:29
        x = B.conv(L['conv12'], [x])
        x = B.conv(L['conv13_upsample'], [B.upsample_nn2x(x)])
        x = B.conv(L['conv14'], [x], post_add=x_1)          # nets.py:32
        x = B.conv(L['conv15_upsample'], [B.upsample_nn2x(x)], post_add=x_0)   # nets.py:33
        x = B.conv(L['conv16'], [x])
        self.logits = B.conv(L['conv17'], [x], outf=mask_out, outf_ch=1, mode=1)   # nets.py:35-41
        return self.logits


def rec_layer_table(f=0.25, C=2):
    """[name, k, cin, cout, stride, identity_act]  (nets.py:57-107)."""
    i = int
    T = []
    for pre, cin0 in (('a', 3), ('b', C + 2)):
        T += [(pre + 'conv1', 7, cin0, i(64 * f), 2, False), (pre + 'conv2', 5, i(64 * f), i(128 * f), 2, False),
              (pre + 'conv3', 5, i(128 * f), i(256 * f), 2, False), (pre + 'conv31', 3, i(256 * f), i(256 * f), 1, False),
              (pre + 'conv4', 3, i(256 * f), i(512 * f), 2, False), (pre + 'conv41', 3, i(512 * f), i(512 * f), 1, False),
              (pre + 'conv5', 3, i(512 * f), i(512 * f), 2, False), (pre + 'conv51', 3, i(512 * f), i(512 * f), 1, False),
              (pre + 'conv6', 3, i(512 * f), i(512 * f), 2, False)]
    T += [('deconv5', 4, i(512 * 2 * f), i(512 * f), 1, False), ('flow5', 3, i(512 * 3 * f), C, 1, True),
          ('deconv4', 4, i(512 * 3 * f), i(512 * f), 1, False), ('upflow4', 4, C, C, 1, True),
          ('flow4', 3, i(512 * 3 * f + C), C, 1, True),
          ('deconv3', 4, i(512 * 3 * f + C), i(256 * f), 1, False), ('upflow3', 4, C, C, 1, True),
          ('flow3', 3, i(256 * 3 * f + C), C, 1, True),
          ('deconv2', 4, i(256 * 3 * f + C), i(128 * f), 1, False), ('upflow2', 4, C, C, 1, True),
          ('flow2', 3, i(128 * 3 * f + C), C, 1, True),
          ('deconv1', 4, i(128 * 3 * f + C), i(64 * f), 1, False), ('upflow1', 4, C, C, 1, True),
          ('flow1', 5, i(64 * 3 * f + C), C, 1, True)]
    return T


class RecoverNet(object):
    """recover_net (nets.py:45-110), batched: the three calls of adversarial_learner.py:114-131 share weights, so the
    b-encoder + decoder run once on a 3B batch and the a-encoder (same image in all three calls) once on B."""

    def __init__(self, store, scope='FlownetS', f=0.25):
        self.scope = scope
        self.layers = {}
        for name, k, cin, cout, s, ident in rec_layer_table(f):
            self.layers[name] = ConvLayer(store, '%s/%s' % (scope, name), k, cin, cout, s, 1, ACT_NONE if ident else ACT_LEAKY, 0.2,
                                          tag='R', wname='weights', bname='biases')

    def all_layers(self):
        return list(self.layers.values())

    def build_a_encoder(self, B, img8):
        """The image encoder depends only on the image: it can be issued early, on the side stream, concurrently with the
        generator (its results are first needed by the decoder concats)."""
        L = self.layers
        d = {}
        x = B.conv(L['aconv1'], [img8]); d['1'] = x
        x = B.conv(L['aconv2'], [x]); d['2'] = x
        x = B.conv(L['aconv3'], [x])
        x = B.conv(L['aconv31'], [x]); d['31'] = x
        x = B.conv(L['aconv4'], [x])
        x = B.conv(L['aconv41'], [x]); d['41'] = x
        x = B.conv(L['aconv5'], [x])
        x = B.conv(L['aconv51'], [x]); d['51'] = x
        x = B.conv(L['aconv6'], [x]); d['6'] = x
        self.a_feats = d
        return d

    def build(self, B, img8, flow_in, flow1_out, ncalls=3):
        """img8: Act [B,H,W,8] (image, 3 real channels); flow_in: Act [ncalls*B,H,W,8] = [flow_masked(2), ones, 1-mask] per call
        (nets.py:50-53); flow1_out: fp32 [ncalls*B,h1,w1,2] receives `flow1` (the final x2 resize is fused into the loss)."""
        L = self.layers
        nB = img8.N
        self._enc = None

        def enc(pre, x):
            d = {}
            x = B.conv(L[pre + 'conv1'], [x]); d['1'] = x
            x = B.conv(L[pre + 'conv2'], [x]); d['2'] = x
            x = B.conv(L[pre + 'conv3'], [x])
            x = B.conv(L[pre + 'conv31'], [x]); d['31'] = x
            x = B.conv(L[pre + 'conv4'], [x])
            x = B.conv(L[pre + 'conv41'], [x]); d['41'] = x
            x = B.conv(L[pre + 'conv5'], [x])
            x = B.conv(L[pre + 'conv51'], [x]); d['51'] = x
            x = B.conv(L[pre + 'conv6'], [x]); d['6'] = x
            return d
        a = self.a_feats if getattr(self, 'a_feats', None) is not None else enc('a', img8)
        b = enc('b', flow_in)
        if ncalls > 1:
            a = {k: v.alias(nB) for k, v in a.items()}
        # `deconv` = legacy-bilinear resize of the concat to the next level + conv: the resize of all concat sources is ONE fused launch
        rs = lambda ts, ref: [B.resize_concat(ts, ref.H, ref.W, name='rs%dx%d' % (ref.H, ref.W))]
        conv6 = [a['6'], b['6']]                                              # nets.py:78
        deconv5 = B.conv(L['deconv5'], rs(conv6, b['51']))
        concat5 = [deconv5, b['51'], a['51']]
        flow5 = B.conv(L['flow5'], concat5)
        deconv4 = B.conv(L['deconv4'], rs(concat5, b['41']))
        upflow4 = B.conv(L['upflow4'], rs([flow5], b['41']))
        concat4 = [deconv4, b['41'], a['41'], upflow4]
        flow4 = B.conv(L['flow4'], concat4)
        deconv3 = B.conv(L['deconv3'], rs(concat4, b['31']))
        upflow3 = B.conv(L['upflow3'], rs([flow4], b['31']))
        concat3 = [deconv3, b['31'], a['31'], upflow3]
        flow3 = B.conv(L['flow3'], concat3)
        deconv2 = B.conv(L['deconv2'], rs(concat3, b['2']))
        upflow2 = B.conv(L['upflow2'], rs([flow3], b['2']))
        concat2 = [deconv2, b['2'], a['2'], upflow2]
        flow2 = B.conv(L['flow2'], concat2)
        deconv1 = B.conv(L['deconv1'], rs(concat2, b['1']))
        upflow1 = B.conv(L['upflow1'], rs([flow2], b['1']))
        concat1 = [deconv1, b['1'], a['1'], upflow1]
        self.flow1 = B.conv(L['flow1'], concat1, outf=flow1_out)
        self.pyramid = dict(flow5=flow5, flow4=flow4, flow3=flow3, flow2=flow2, flow1=self.flow1)
        return self.flow1


def generator_net(images, flows, scope='MaskNet', reuse=None, training=True, params=None):
    """Function-level API of the reference (nets.py:4-42); see models/functional.py."""
    from . import functional
    return functional.generator_net(images, flows, scope, reuse, training, params)


def recover_net(img1, flow_masked, mask, scope='FlownetS', reuse=None, f=0.25, training=True, params=None):
    """Function-level API of the reference (nets.py:45-110); see models/functional.py."""
    from . import functional
    return functional.recover_net(img1, flow_masked, mask, scope, reuse, f, training, params)
