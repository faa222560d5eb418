"""Launch census of the PWC-Net training step (FlowTrainGraph) without a GPU: the graphs of tests/test_flow_train_launches_gpu.py are
BUILT on CPU tensors (nothing is launched) and checked for what the GPU walk relies on.

  default   FlowTrainGraph(192, 384, 16, in_hw=(384, 640)): train_flow.py's defaults on one GPU, multi-scale loss
  unsup     the same with loss='unsupervised': network batch 32
  timed     FlowTrainGraph(384, 640, 8): tools/time_flow_train.py's timed step
  shard     FlowTrainGraph(192, 384, 4, global_batch=16, in_hw=(384, 640), loss='robust', options={'use_dense_cx': False},
            augment=True, sample_offset=8): the robust loss, the "sm" network, the augmentation, rank 2 of 4

Every op of the aug, fwd, bwd, adam and pack plans has exactly one owner, the glue and conv launch counts are pinned, and so are the
arguments that motivate each graph, so that a builder change which silently stops exercising one of them fails here.  The ratchet: every
entry point of the C ABI binding is owned by a per-launch check or listed in FUNCTION_LEVEL with the test file that checks it, and no
plan of any graph of the three CPU launch-census files (this one, tests/test_glue_launches_cpu.py, tests/test_graph_variants_launches_cpu.py)
launches a listed one.  The next kernel added to a step without a per-launch reference fails here."""
import collections
import os

import pytest
import torch

import conv_launch_ref as R
import glue_launch_ref as G
import unsup_flow_loss_ref as UR
from unsupervised_detection_b200 import _lib
from unsupervised_detection_b200.flow_train_graph import ALPHAS, LEVELS, FlowTrainGraph
from unsupervised_detection_b200.models.PWCNet.model_pwcnet import FLOW_PRED_LVL
from test_conv_launches_cpu import _attributed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLANS = ('aug', 'fwd', 'bwd', 'adam', 'pack')
GRAPHS = {
    'default': ((192, 384, 16), dict(in_hw=(384, 640))),
    'unsup': ((192, 384, 16), dict(in_hw=(384, 640), loss='unsupervised')),
    'timed': ((384, 640, 8), {}),
    'shard': ((192, 384, 4), dict(global_batch=16, in_hw=(384, 640), loss='robust', options={'use_dense_cx': False}, augment=True,
                                  sample_offset=8)),
}
KEYS = list(GRAPHS)

# glue launches per plan
_BWD = {'cis_zero': 5, 'cis_flow_multiscale_loss_bwd': 1, 'cis_colsum': 18, 'cis_dact_colsum': 91, 'cis_warp_costvol_bwd': 5,
        'cis_parity_split_bf16': 8}
_FWD = {'cis_resize_bilinear_f32': 3, 'cis_pack_f32_to_bf16': 2, 'cis_warp_costvol': 5, 'cis_flow_multiscale_loss': 1}
_ADAM = {'cis_adam_l2': 1}
DEFAULT = {'aug': {}, 'fwd': _FWD, 'bwd': _BWD, 'adam': _ADAM, 'pack': {}}
GLUE = {
    'default': DEFAULT,
    'unsup': dict(DEFAULT, fwd={'cis_resize_bilinear_f32': 3, 'cis_pack_f32_to_bf16': 4, 'cis_warp_costvol': 5, 'cis_unsup_flow_loss': 1},
                  bwd=dict({k: v for k, v in _BWD.items() if k != 'cis_flow_multiscale_loss_bwd'}, cis_unsup_flow_loss_bwd=1,
                           cis_resize_f32_bwd_to_bf16_scaled=1)),
    'timed': dict(DEFAULT, fwd=dict(_FWD, cis_resize_bilinear_f32=1)),     # no input resize: only the final x4
    'shard': dict(DEFAULT, aug={'cis_flow_aug_params': 1, 'cis_flow_augment': 1}),
}
# conv launches (cis_conv_igemm + cis_conv_wgrad) of fwd + bwd
CONV = {'default': 367, 'unsup': 367, 'timed': 355, 'shard': 367}

# Entry points no launch plan of the checked graphs uses: each is checked against fp64 at the function level, by the file named.  The
# groups say how that file reaches them; a file that stops reaching its entry points this way must be replaced here.
FUNCTION_LEVEL = {
    # called by name, on buffers the test builds
    'cis_abs_sum': 'tests/test_flow_train_launches_gpu.py', 'cis_crop_resize_flow_f32': 'tests/test_flow_train_launches_gpu.py',
    'cis_masked_epe': 'tests/test_flow_train_launches_gpu.py',          # these two through FlowTrainGraph.epe()
    'cis_crop_resize_bilinear_f32': 'tests/test_kernels_gpu.py', 'cis_dense_image_warp': 'tests/test_kernels_gpu.py',
    'cis_resize_nn_f32': 'tests/test_kernels_gpu.py', 'cis_cost_volume_bwd_r': 'tests/test_pwc_options_gpu.py',
    # the parameter-space ops: planned by name, batched into cis_param_multi jobs (Plan.batch_param_ops).  The conv references read
    # bf16 of the fp32 master (the packs), the weight- and bias-gradient checks read the stored gradients (the un-pack and the BN chain
    # rule), and check_bn_fold compares the folded weights (the BN fold)
    'cis_bn_chain': 'tests/test_conv_launches_gpu.py', 'cis_bn_fold': 'tests/test_conv_launches_gpu.py',
    'cis_pack_weights': 'tests/test_conv_launches_gpu.py', 'cis_pack_weights_tiled': 'tests/test_conv_launches_gpu.py',
    'cis_unpack_wgrad': 'tests/test_conv_launches_gpu.py',
    # the function-level API (models/functional.py): the wrappers' forward and backward against the fp64 oracle
    'cis_charbonnier_sum': 'tests/test_functional_api_gpu.py',                                         # charbonnier_loss
    'cis_charbonnier_bwd': 'tests/test_functional_grad_gpu.py', 'cis_cost_volume_bwd': 'tests/test_functional_grad_gpu.py',
    'cis_dense_image_warp_bwd': 'tests/test_functional_grad_gpu.py',
    'cis_cast_bf16_to_f32_scaled': 'tests/test_functional_grad_gpu.py',                                 # recover_net's mask gradient
    'cis_cast_f32_to_bf16': 'tests/test_layer_api_gpu.py',                                              # the layer cells' input and seed
    'cis_flow_standardize': 'tests/test_layer_api_gpu.py', 'cis_flow_standardize_bwd': 'tests/test_layer_api_gpu.py',   # preprocess_flow_batch
    'cis_resize_f32': 'tests/test_layer_api_gpu.py', 'cis_resize_f32_bwd': 'tests/test_layer_api_gpu.py',           # the resize modes
}


def build(key, device):
    """(FlowTrainGraph, conv Recorder, [(plan name, Plan)]) of one of KEYS."""
    a, kw = GRAPHS[key]
    mp = pytest.MonkeyPatch()
    with R.recorded(mp) as rec:
        g = FlowTrainGraph(*a, device=device, **kw)
    return g, rec, [(p, getattr(g, p)) for p in PLANS]


@pytest.fixture(scope='module')
def graphs():
    return {k: build(k, 'cpu') for k in KEYS}


def _ops(graphs, key, plan):
    return [op for name, p in graphs[key][2] if name == plan for op in p.ops]


@pytest.mark.parametrize('key', KEYS)
def test_every_launch_has_one_owner(graphs, key):
    owners = [set(G.ARGS), G.CONV_WALKER, set(G.PINNED_ELSEWHERE), G.STRUCTURAL]
    for name, plan in graphs[key][2]:
        for op in plan.ops:
            assert sum(op[2] in s for s in owners) == 1, (key, name, op[2])


@pytest.mark.parametrize('key', KEYS)
def test_glue_launch_counts(graphs, key):
    plans = dict(graphs[key][2])
    assert set(plans) == set(GLUE[key])
    for name, plan in plans.items():
        assert dict(G.glue_counts(plan)) == GLUE[key][name], (key, name)
        for op in plan.ops:
            if op[2] in G.ARGS:
                G.decode(op)


@pytest.mark.parametrize('key', KEYS)
def test_every_conv_op_is_attributed_once(graphs, key):
    plans = [p for _, p in graphs[key][2]]
    checks = _attributed(graphs[key][1], plans)
    assert sum(len(R.conv_ops(p)) for p in plans) == sum(len(ck.ops) for ck in checks) == CONV[key]


def test_default_geometry_resizes_the_frames_and_scales_the_targets(graphs):
    """384x640 uploads, a 192x384 network: both frames and the final x4 go through cis_resize_bilinear_f32, and the loss samples the
    targets with the vector scales s0 = 192/384, s1 = 384/640."""
    g = graphs['default'][0]
    res = [G.decode(op) for op in _ops(graphs, 'default', 'fwd') if op[2] == 'cis_resize_bilinear_f32']
    assert [(r['H'], r['W'], r['OH'], r['OW'], r['C'], r['scale']) for r in res] == \
        [(384, 640, 192, 384, 3, 1.0)] * 2 + [(48, 96, 192, 384, 2, 4.0)]
    for plan, name in (('fwd', 'cis_flow_multiscale_loss'), ('bwd', 'cis_flow_multiscale_loss_bwd')):
        a = [G.decode(op) for op in _ops(graphs, 'default', plan) if op[2] == name][0]
        assert (a['B'], a['H'], a['W'], a['GH'], a['GW'], a['robust']) == (16, 192, 384, 384, 640, 0)
        assert float(G._f32(a['s0'])) == 0.5 and float(G._f32(a['s1'])) == float(G._f32(0.6))
        assert a['gt'] == g.batch[2].data_ptr()


def test_level_weights_of_the_sharded_graph(graphs):
    """Rank 2 of 4: weight alpha_l / global batch, the robust rho, the augmented ground truth, and its sample offset."""
    g = graphs['shard'][0]
    a = [G.decode(op) for op in _ops(graphs, 'shard', 'fwd') if op[2] == 'cis_flow_multiscale_loss'][0]
    pyr = a['pyr']._obj
    assert [pyr.weight[i] for i in range(5)] == [float(G._f32(al / 16)) for al in ALPHAS]
    assert (a['robust'], a['B'], a['gt']) == (1, 4, g.batch[2].data_ptr()) and g.batch[2].data_ptr() != g.gt.data_ptr()
    p = [G.decode(op) for op in _ops(graphs, 'shard', 'aug') if op[2] == 'cis_flow_aug_params'][0]
    assert (p['B'], p['H'], p['W'], p['sample_offset'], p['step']) == (4, 384, 640, 8, g.step_state.data_ptr())


def test_unsupervised_packs_and_seed(graphs):
    """The four packs: each image Act holds both frames, the second of each pair at +half and swapped; the seed's weights are
    1 / (GB H W) and lambda / (GB H W), and the final x4 resize's transpose seeds the level-2 flow gradient with scale 4."""
    g = graphs['unsup'][0]
    B, H, W = 16, 192, 384
    frames = [G.decode(op)['dst'] for op in _ops(graphs, 'unsup', 'fwd') if op[2] == 'cis_resize_bilinear_f32'][:2]
    packs = [G.decode(op) for op in _ops(graphs, 'unsup', 'fwd') if op[2] == 'cis_pack_f32_to_bf16']
    i1, i2 = g.img_acts
    half = B * H * W * i1.pitch * 2
    assert [(p['src'], p['dst'], p['npix'], p['offset']) for p in packs] == [
        (frames[0], i1.ptr, B * H * W, 0.5), (frames[1], i1.ptr + half, B * H * W, 0.5),
        (frames[1], i2.ptr, B * H * W, 0.5), (frames[0], i2.ptr + half, B * H * W, 0.5)]
    bwd = _ops(graphs, 'unsup', 'bwd')
    lb = [G.decode(op) for op in bwd if op[2] == 'cis_unsup_flow_loss_bwd'][0]
    assert float(G._f32(lb['w_photo'])) == float(G._f32(1.0 / (B * H * W)))
    assert float(G._f32(lb['w_smooth'])) == float(G._f32(3.0 / (B * H * W)))
    sd = [G.decode(op) for op in bwd if op[2] == 'cis_resize_f32_bwd_to_bf16_scaled'][0]
    fg = g.pwc.flows_bf[FLOW_PRED_LVL].get_grad()
    assert FLOW_PRED_LVL == 2 and (sd['dd'], sd['N'], sd['ds'], sd['scale'], sd['H'], sd['W']) == (lb['dflow'], 2 * B, fg.ptr, 4.0, H // 4, W // 4)


@pytest.mark.parametrize('key,accumulate', [('default', True), ('unsup', False)])
def test_level_gradient_accumulation(graphs, key, accumulate):
    """Multi-scale: the loss backward overwrites all five level-flow gradients (pyr.accumulate = 0), then up_flow's data gradient adds
    into levels 3-6.  Unsupervised: no loss backward at those levels, and up_flow's data gradient writes them."""
    g, rec = graphs[key][0], graphs[key][1]
    if key == 'default':
        a = [G.decode(op) for op in _ops(graphs, key, 'bwd') if op[2] == 'cis_flow_multiscale_loss_bwd'][0]
        pyr = a['pyr']._obj
        assert list(pyr.accumulate) == [0] * 5
        assert [pyr.grad[i] for i in range(5)] == [g.pwc.flows_bf[l].get_grad().ptr for l in LEVELS]
    for l in (3, 4, 5, 6):
        gr = g.pwc.flows_bf[l].get_grad()
        cks = [ck for ck in rec.checks if ck.kind == 'dgrad' and ck.info['tgt'] is gr]
        assert len(cks) == 1 and cks[0].layer.name == 'pwcnet/upsample/up_flow%d' % l
        d = cks[0].descs()[0]
        assert d.out == gr.ptr and (d.add_pre == gr.ptr) == accumulate and (bool(d.add_pre) == accumulate), (l, d.add_pre)


# ------------------------------------------------------------------------------------------------ the ratchet
def test_every_entry_point_is_owned_or_listed():
    owned = set(G.ARGS) | G.CONV_WALKER | set(G.PINNED_ELSEWHERE)
    assert not owned & set(FUNCTION_LEVEL), owned & set(FUNCTION_LEVEL)
    missing = sorted(set(_lib._PROTOS) - owned - set(FUNCTION_LEVEL))
    assert not missing, 'entry points with neither a per-launch reference nor a function-level test: %s' % missing
    assert set(FUNCTION_LEVEL) <= set(_lib._PROTOS)
    for name, path in FUNCTION_LEVEL.items():
        assert os.path.isfile(os.path.join(ROOT, path)), (name, path)


def test_no_checked_graph_launches_a_function_level_entry_point(graphs):
    import test_glue_launches_cpu as GC
    import test_graph_variants_launches_cpu as GV
    from unsupervised_detection_b200.models import functional as FN
    plans = [(k, n, p) for k, (_, _, ps) in graphs.items() for n, p in ps]
    for key, args, kw in (('config2', (256, 448, 4), {}), ('defaults', (192, 384, 16), dict(with_pwc=False)),
                          ('odd', (100, 172, 3), dict(with_pwc=False)), ('boxes', (256, 448, 4), dict(masks='boxes'))):
        plans += [(key, n, p) for n, p in GC._graph(*args, **kw)[1].items()]
    r = FN._PWCRunner(2, 384, 640, 'cpu', 'pwcnet', trainable=True)
    r.ensure_backward()
    plans += [('pwc_runner', 'fwd', r.bld.fwd), ('pwc_runner', 'bwd', r.bwd)]
    for key in GV.KEYS:
        plans += [(key, n, p) for n, p in GV.build(key, 'cpu')[2]]
    for key, name, plan in plans:
        for op in plan.ops:
            assert op[2] not in FUNCTION_LEVEL, (key, name, op[2])


# ------------------------------------------------------------------------------------------------ the backward gather restated
def test_unsup_bwd_gather_is_autograd_of_the_loss():
    """glue_launch_ref.unsup_bwd_gather (the reference of cis_unsup_flow_loss_bwd: the folded census window through dense_image_warp's
    dflow rule, plus the 5-point smoothness stencil) against autograd of unsup_flow_loss_ref.loss with the mask held fixed."""
    gen = torch.Generator().manual_seed(31)
    B, H, W = 2, 11, 14
    D = torch.float64
    i1 = torch.rand(B, H, W, 3, generator=gen, dtype=D) - 0.5
    i2 = torch.rand(B, H, W, 3, generator=gen, dtype=D) - 0.5
    flow = torch.randn(2 * B, H, W, 2, generator=gen, dtype=D) * 1.5
    GB, lam = 3, 2.0
    M = UR.mask(flow)[0]
    fr = flow.clone().requires_grad_(True)
    (ref,) = torch.autograd.grad(UR.loss(fr, i1, i2, global_batch=GB, smooth_weight=lam, m=M), fr)
    _, t = UR.direction_sums(flow, i1, i2, m=M)
    coef = M * 0.4 * (t['c'] + 0.01) ** -0.6
    got = G.unsup_bwd_gather(flow, i1, i2, t['warped'], coef, 1.0 / (GB * H * W), lam / (GB * H * W), bounds=True)
    assert torch.allclose(got['ref'], ref, rtol=1e-10, atol=1e-14)
    assert bool((got['smooth'] != 0).any()) and bool((got['photo'] != 0).any())
    assert bool(torch.isfinite(got['err']).all()) and bool((got['err'] > 0).all())
