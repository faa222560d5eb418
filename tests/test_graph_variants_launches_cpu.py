"""Per-launch coverage of the graphs the project ships besides the three of tests/test_conv_launches_gpu.py, without a GPU: the graphs of
tests/test_graph_variants_launches_gpu.py are BUILT on CPU tensors (nothing is launched) and checked for what the GPU file relies on.

  gen_fwd     CISGraph(128, 224, 1, with_pwc=False, train=False): bench.py --workload gen_fwd, test_generator.py
  ensemble    CISGraph(192, 384, 4, train=False), the default PWC-Net options: bench.py --workload ensemble, the 4-crop ensemble
  odd         CISGraph(100, 172, 3, with_pwc=False), train: any size that is not a multiple of 64 (partial 16 x 8 tiles, odd widths)
  r1, r2, r3  _PWCRunner(2, 384, 640, trainable=True, options={'search_range': r}), forward and backward
  dense_off   the same with use_dense_cx=False (the "sm" checkpoints)

The two inference graphs are walked as their mask plan (_mask_plan: what forward_masks and the benchmark run) followed by the rest of
the forward; the two parts hold every forward op once.  Every conv op is attributed to exactly one check, every entry point has one
owner (conv walker, glue reference table, a test that pins it elsewhere, structural op), the glue launch counts per plan are pinned, and
the configurations that motivate these checks must still be there, so a planner change that silently stops exercising one fails here."""
import collections
import ctypes as C

import pytest

import conv_launch_ref as R
import glue_launch_ref as G
from launch_suites import CONV, GLUE, VARIANTS, attributed, build, features
from unsupervised_detection_b200 import _lib
from unsupervised_detection_b200.models.PWCNet.model_pwcnet import A_TOTAL, CORR_OFF


@pytest.fixture(scope='module')
def graphs():
    return {k: build(k, 'cpu') for k in VARIANTS}


def _checks(graphs, key):
    return attributed(graphs[key][1], [p for _, p in graphs[key][2]])


@pytest.mark.parametrize('key', VARIANTS)
def test_every_conv_op_is_attributed_once(graphs, key):
    checks = _checks(graphs, key)
    assert sum(len(R.conv_ops(p)) for _, p in graphs[key][2]) == sum(len(ck.ops) for ck in checks) == CONV[key]


@pytest.mark.parametrize('key', VARIANTS)
def test_every_launch_has_one_owner(graphs, key):
    owners = [set(G.ARGS), G.CONV_WALKER, set(G.PINNED_ELSEWHERE), G.STRUCTURAL]
    for name, plan in graphs[key][2]:
        for op in plan.ops:
            assert sum(op[2] in s for s in owners) == 1, (key, name, op[2])


@pytest.mark.parametrize('key', VARIANTS)
def test_glue_launch_counts(graphs, key):
    plans = dict(graphs[key][2])
    want = GLUE[key]
    assert set(plans) == set(want)
    for name, plan in plans.items():
        assert dict(G.glue_counts(plan)) == want[name], (key, name)
        for op in plan.ops:
            if op[2] in G.ARGS:
                G.decode(op)


def test_range1_conv6_0_is_a_compact_16_channel_launch_on_9_channels(graphs):
    """predict_flow/conv6_0 at search range 1 reads the 9-channel cost volume, padded to 16, through the compact thin = 16 format."""
    cks = [ck for ck in _checks(graphs, 'r1') if ck.kind == 'fwd' and ck.layer.name == 'pwcnet/predict_flow/conv6_0']
    assert len(cks) == 1
    d, src = cks[0].descs()[0], cks[0].info['srcs']
    assert d.halo == 1 and d.thin == 16 and cks[0].layer.cin == 9
    assert len(src) == 1 and [m >= 0 for m in src[0].chanmap] == [True] * 9 + [False] * 7


@pytest.mark.parametrize('key,r,pad', [('r1', 1, 16), ('r2', 2, 32), ('r3', 3, 56)])
def test_cost_volume_range_launches(graphs, key, r, pad):
    """Every warp + cost-volume launch of a range-r network takes the _r entry point with range r, and writes the (2r+1)^2 channels at
    the corr slice, whose padding up to `pad` channels the level buffer's views mark as padding."""
    net = graphs[key][0].net
    assert (net.ndisp, net.corr_pad, net.c1_off) == ((2 * r + 1) ** 2, pad, CORR_OFF + pad)
    pitches = {net.level_pitch(l) for l in range(2, 7)}
    n = collections.Counter()
    for name, plan in graphs[key][2]:
        for op in plan.ops:
            if op[2].startswith('cis_warp_costvol'):
                a = G.decode(op)
                pitch, off = (a['op'], a['oo']) if op[2] == 'cis_warp_costvol_r' else (a['dcp'], a['dco'])
                assert a['r'] == r and pitch in pitches and off == CORR_OFF, op[2]
                n[op[2]] += 1
    assert n == {'cis_warp_costvol_r': 5, 'cis_warp_costvol_bwd_r': 5}
    for l in range(2, 7):
        assert [m >= 0 for m in net._chanmap(l, A_TOTAL)[:pad]] == [True] * net.ndisp + [False] * (pad - net.ndisp)


def test_ensemble_recover_split_k_over_batch_broadcast_concats(graphs):
    """The recover net of the ensemble runs at N = 12 (three calls of 4 crops); its flow heads read 3- and 4-source concats whose
    batch-broadcast sources repeat, split 6 and 7 ways over K."""
    f = features(_checks(graphs, 'ensemble'))
    assert {('n_mod', 3, 6), ('n_mod', 4, 7)} <= f, sorted(x for x in f if isinstance(x, tuple) and x[0] == 'n_mod')
    big = [ck for ck in _checks(graphs, 'ensemble') if ck.layer.name.startswith('FlownetS/') and ck.descs()[0].splits >= 6
           and ck.descs()[0].nsrc == 4]
    assert big and all(ck.descs()[0].N == 12 for ck in big)


def test_odd_graph_partial_tiles_in_every_launch_kind(graphs):
    """100 x 172: output grids whose width is not a multiple of 8 and whose height is not a multiple of 16, in the forward, the data
    gradient and the weight gradient."""
    kinds = collections.Counter(ck.kind for ck in _checks(graphs, 'odd') for d in ck.descs() if d.OW % 8 and d.OH % 16)
    assert kinds['fwd'] > 0 and kinds['dgrad'] > 0 and kinds['wgrad'] > 0, kinds


def _s2_phase(d):
    h, wk = _lib.CisConv(), (C.c_int16 * (2 * 49))()
    return bool(_lib.load().cis_conv_s2_phase_plan(C.byref(d), C.byref(h), wk))


def test_ensemble_stride2_phase_halo_launches(graphs):
    """The stride-2 forward launches cis_conv_igemm rewrites into compact phase-halo launches (cis_conv_s2_phase_plan): PWC-Net's first
    two pyramid levels for both frames and the recover encoders' first layers."""
    names = collections.Counter(ck.layer.name for ck in _checks(graphs, 'ensemble')
                                if ck.kind == 'fwd' and not ck.descs()[0].halo and ck.layer.stride == 2 and _s2_phase(ck.descs()[0]))
    assert names['pwcnet/featpyr/conv1a'] == 2 and names['pwcnet/featpyr/conv2a'] == 2, names
    assert {'FlownetS/aconv1', 'FlownetS/bconv1'} <= set(names), names
