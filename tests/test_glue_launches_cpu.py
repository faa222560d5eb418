"""Ownership of every launch of the benchmarked graphs, without a GPU: the graphs of tests/test_glue_launches_gpu.py are BUILT on CPU
tensors (nothing is launched), and every entry point in their forward and backward plans must have exactly one owner -- the conv walker,
the glue checker's reference table (tests/glue_launch_ref.py), a test that pins it elsewhere, or the structural ops.  A kernel added to
the step without a per-launch reference fails here.  The per-graph launch counts of the GPU checks are pinned too."""
import collections

import pytest

import glue_launch_ref as G
from unsupervised_detection_b200 import _lib
from unsupervised_detection_b200.models import functional as FN
from unsupervised_detection_b200.step_graph import CISGraph

CONFIG2 = {
    'fwd': {'cis_resize_concat_bf16': 11, 'cis_warp_costvol': 5, 'cis_pack_f32_to_bf16': 3, 'cis_resize_bilinear_f32': 3,
            'cis_upsample_nn2x': 2, 'cis_flow_stats': 1, 'cis_pack_generator_input': 1, 'cis_zero': 2},
    'bwd_R': {'cis_dact_colsum': 23, 'cis_resize_concat_bf16_bwd': 14, 'cis_colsum': 9},
    'bwd_G': {'cis_dact_colsum': 16, 'cis_dact_mul': 14, 'cis_resize_concat_bf16_bwd': 14, 'cis_add_slice': 3, 'cis_upsample_nn2x_bwd': 2,
              'cis_colsum': 1},
}
PWC_BWD = {'cis_dact_colsum': 91, 'cis_colsum': 18, 'cis_parity_split_bf16': 8, 'cis_warp_costvol_bwd': 5, 'cis_zero': 5,
           'cis_cast_bf16_to_f32': 2, 'cis_resize_f32_bwd_to_bf16_scaled': 1}
PWC_FWD = {'cis_warp_costvol': 5, 'cis_pack_f32_to_bf16': 2, 'cis_resize_bilinear_f32': 1}
# the flow given directly: no PWC-Net, no 384x640 inputs
FLOW_GIVEN = dict(CONFIG2, fwd={'cis_resize_concat_bf16': 11, 'cis_pack_f32_to_bf16': 1, 'cis_upsample_nn2x': 2, 'cis_flow_stats': 1,
                                'cis_pack_generator_input': 1, 'cis_zero': 2})
BOXES = {'fwd': {'cis_resize_concat_bf16': 11, 'cis_warp_costvol': 5, 'cis_pack_f32_to_bf16': 3, 'cis_resize_bilinear_f32': 3, 'cis_zero': 1},
         'bwd_R': CONFIG2['bwd_R']}


def _graph(*a, **k):
    g = CISGraph(*a, device='cpu', **k)
    plans = {'fwd': g.fwd}
    plans.update({'bwd_' + m: p for m, p in g.bwd.items()})
    return g, plans


@pytest.fixture(scope='module')
def graphs():
    r = FN._PWCRunner(2, 384, 640, 'cpu', 'pwcnet', trainable=True)
    r.ensure_backward()
    out = {'config2': _graph(256, 448, 4), 'defaults': _graph(192, 384, 16, with_pwc=False), 'odd': _graph(100, 172, 3, with_pwc=False),
           'boxes': _graph(256, 448, 4, masks='boxes'), 'pwc_runner': (r, {'fwd': r.bld.fwd, 'bwd': r.bwd})}
    return out


def test_owner_sets_are_disjoint():
    sets = [set(G.ARGS), G.CONV_WALKER, set(G.PINNED_ELSEWHERE), G.STRUCTURAL]
    for i in range(len(sets)):
        for j in range(i + 1, len(sets)):
            assert not sets[i] & sets[j], sets[i] & sets[j]


@pytest.mark.parametrize('key', ['config2', 'defaults', 'odd', 'boxes', 'pwc_runner'])
def test_every_launch_has_one_owner(graphs, key):
    owners = set(G.ARGS) | G.CONV_WALKER | set(G.PINNED_ELSEWHERE) | G.STRUCTURAL
    for name, plan in graphs[key][1].items():
        for op in plan.ops:
            assert op[2] in owners, (key, name, op[2])


def test_references_decode_the_abi():
    """Each reference names as many arguments as the binding declares, and every glue op of the graphs passes that many."""
    for name, spec in G.ARGS.items():
        assert len(spec.split()) == len(_lib._PROTOS[name]), name
        assert name in _lib._PROTOS


@pytest.mark.parametrize('key,want', [('config2', CONFIG2), ('defaults', FLOW_GIVEN), ('odd', FLOW_GIVEN), ('boxes', BOXES),
                                      ('pwc_runner', {'fwd': PWC_FWD, 'bwd': PWC_BWD})])
def test_glue_launch_counts(graphs, key, want):
    plans = graphs[key][1]
    assert set(plans) == set(want)
    for name, plan in plans.items():
        assert dict(G.glue_counts(plan)) == want[name], (key, name)
        for op in plan.ops:
            if op[2] in G.ARGS:
                G.decode(op)


def test_odd_geometry_runs_the_generic_resize():
    """100x172: the recover decoder's 4x6 -> 7x11 -> 13x22 -> 25x43 resize-concats take the generic (non-x2) kernel and transpose."""
    _, plans = _graph(100, 172, 3, with_pwc=False)
    kinds = collections.Counter()
    for name, plan in plans.items():
        for op in plan.ops:
            if op[2].startswith('cis_resize_concat_bf16'):
                a = G.decode(op)
                kinds[(name, G.Glue._rc_kind(a['H'], a['W'], a['OH'], a['OW']))] += 1
    assert kinds[('fwd', 'generic')] == 6 and kinds[('bwd_R', 'generic')] == 6 and kinds[('bwd_G', 'generic')] == 6, kinds
