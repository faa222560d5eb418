"""Reference PWC-Net for every option set the package supports (use_dense_cx, use_res_cx, search_range), composed from the unchanged
oracle primitives (oracle/pwcnet.py: cost_volume, dense_image_warp, extract_features, refine_flow; oracle/tf_ops.py).  With the default
options every function here computes exactly what oracle.pwcnet / oracle.params compute (test_pwc_options_cpu.py checks that).

Option semantics follow models/PWCNet/model_pwcnet.py of the reference: predict_flow :476-506 (`x = concat([act, x])` only with dense
connections, otherwise `x = act`), nn :606-642 (refine_flow above the prediction level only with use_res_cx, always at it)."""
import math

import torch

from oracle import params as OP, pwcnet as PW, tf_ops as T

LG = {'search_range': 4, 'use_dense_cx': True, 'use_res_cx': True}
DENSE = (128, 128, 96, 64, 32)
CTX = (128, 128, 128, 96, 64, 32, 2)


def opts(options=None):
    o = dict(LG)
    o.update({k: v for k, v in (options or {}).items() if k in LG})
    return o


def pwc_layers(options=None):
    """names -> (k, cin, cout, transposed), in the order of oracle.params.pwc_layers."""
    o = opts(options)
    nd = (2 * o['search_range'] + 1) ** 2
    nc = PW.NUM_CHANN
    L = []
    cin = 3
    for l in range(1, 7):
        L += [(f'featpyr/conv{l}a', 3, cin, nc[l], False), (f'featpyr/conv{l}aa', 3, nc[l], nc[l], False),
              (f'featpyr/conv{l}b', 3, nc[l], nc[l], False)]
        cin = nc[l]
    for l in range(6, 1, -1):
        c = nd if l == 6 else nd + nc[l] + 4
        for i, co in enumerate(DENSE):
            L.append((f'predict_flow/conv{l}_{i}', 3, c, co, False))
            c = c + co if o['use_dense_cx'] else co
        L.append((f'predict_flow/flow{l}', 3, c, 2, False))
        if o['use_res_cx'] or l == 2:
            cc = c
            for i, co in enumerate(CTX, start=1):
                L.append((f'ctxt/dc_conv{l}{i}', 3, cc, co, False))
                cc = co
        if l != 2:
            L.append((f'upsample/up_flow{l}', 4, 2, 2, True))
            L.append((f'upsample/up_feat{l}', 4, c, 2, True))
    return L


def param_count(options=None):
    return sum(k * k * ci * co + co for _, k, ci, co, _ in pwc_layers(options))


def make_params(seed=8964, dtype=torch.float32, jitter=0.0, options=None):
    """oracle.params.make_params(nets=('pwcnet',)) for the option set's layer table (same generator sequence, same initialisers)."""
    g = torch.Generator().manual_seed(seed)
    p = {}
    jit = lambda n: (torch.rand(n, generator=g, dtype=dtype) * 2 - 1) * jitter
    for name, k, cin, cout, tr in pwc_layers(options):
        if tr:
            lim = math.sqrt(6.0 / (k * k * cout + k * k * cin))
            p[f'pwcnet/{name}/kernel'] = (torch.rand(k, k, cout, cin, generator=g, dtype=dtype) * 2 - 1) * lim
        else:
            std = math.sqrt(2.0 / (k * k * cin))
            p[f'pwcnet/{name}/kernel'] = torch.randn(k, k, cin, cout, generator=g, dtype=dtype) * std
        p[f'pwcnet/{name}/bias'] = jit(cout)
    return p


def predict_flow(corr, c1, up_flow, up_feat, lvl, p, dense=True):
    x = corr if c1 is None else torch.cat([corr, c1, up_flow, up_feat], 3)
    for i in range(5):
        act = PW._c(x, p, f'pwcnet/predict_flow/conv{lvl}_{i}')
        x = torch.cat([act, x], 3) if dense else act
    return x, PW._c(x, p, f'pwcnet/predict_flow/flow{lvl}', act=False)


def predict_from_img_pairs(img1, img2, p, return_pyr=False, options=None):
    """oracle.pwcnet.predict_from_img_pairs for an option set."""
    o = opts(options)
    r = o['search_range']
    c1 = PW.extract_features(img1 + 0.5, p)
    c2 = PW.extract_features(img2 + 0.5, p)
    flow_pyr = []
    up_flow = up_feat = None
    for lvl in range(6, 1, -1):
        if lvl == 6:
            corr = PW.cost_volume(c1[lvl], c2[lvl], r)
            upfeat, flow = predict_flow(corr, None, None, None, lvl, p, o['use_dense_cx'])
        else:
            warp = PW.dense_image_warp(c2[lvl], up_flow * (20.0 / 2 ** lvl))
            corr = PW.cost_volume(c1[lvl], warp, r)
            upfeat, flow = predict_flow(corr, c1[lvl], up_flow, up_feat, lvl, p, o['use_dense_cx'])
        if o['use_res_cx'] or lvl == 2:
            flow = PW.refine_flow(upfeat, flow, lvl, p)
        flow_pyr.append(flow)
        if lvl != 2:
            up_flow = T.conv2d_transpose_k4s2(flow, p[f'pwcnet/upsample/up_flow{lvl}/kernel'], p[f'pwcnet/upsample/up_flow{lvl}/bias'])
            up_feat = T.conv2d_transpose_k4s2(upfeat, p[f'pwcnet/upsample/up_feat{lvl}/kernel'], p[f'pwcnet/upsample/up_feat{lvl}/bias'])
        else:
            flow_pred = T.resize_bilinear_legacy(flow, flow.shape[1] * 4, flow.shape[2] * 4) * 4
    if return_pyr:
        return flow_pred, flow_pyr, c1, c2
    return flow_pred


def default_tables_match_oracle():
    return pwc_layers() == OP.pwc_layers()
