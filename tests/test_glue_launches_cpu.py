"""Ownership of every launch of the benchmarked graphs, without a GPU: the graphs tests/test_conv_launches_gpu.py and
tests/test_glue_launches_gpu.py check are BUILT on CPU tensors (nothing is launched), and every entry point in their forward and backward
plans must have exactly one owner -- the conv walker, the glue checker's reference table (tests/glue_launch_ref.py), a test that pins it
elsewhere, or the structural ops.  A kernel added to the step without a per-launch reference fails here.  The per-graph launch counts of
the GPU checks are pinned too."""
import collections

import pytest

import glue_launch_ref as G
from launch_suites import GLUE, build
from unsupervised_detection_b200 import _lib

KEYS = ['config2', 'defaults', 'odd', 'boxes', 'pwc_runner']


@pytest.fixture(scope='module')
def graphs():
    return {k: dict(build(k, 'cpu')[2]) for k in KEYS}


def test_owner_sets_are_disjoint():
    sets = [set(G.ARGS), G.CONV_WALKER, set(G.PINNED_ELSEWHERE), G.STRUCTURAL]
    for i in range(len(sets)):
        for j in range(i + 1, len(sets)):
            assert not sets[i] & sets[j], sets[i] & sets[j]


@pytest.mark.parametrize('key', KEYS)
def test_every_launch_has_one_owner(graphs, key):
    owners = set(G.ARGS) | G.CONV_WALKER | set(G.PINNED_ELSEWHERE) | G.STRUCTURAL
    for name, plan in graphs[key].items():
        for op in plan.ops:
            assert op[2] in owners, (key, name, op[2])


def test_references_decode_the_abi():
    """Each reference names as many arguments as the binding declares, and every glue op of the graphs passes that many."""
    for name, spec in G.ARGS.items():
        assert len(spec.split()) == len(_lib._PROTOS[name]), name
        assert name in _lib._PROTOS


@pytest.mark.parametrize('key,want', [(k, GLUE[k]) for k in KEYS])
def test_glue_launch_counts(graphs, key, want):
    plans = graphs[key]
    assert set(plans) == set(want)
    for name, plan in plans.items():
        assert dict(G.glue_counts(plan)) == want[name], (key, name)
        for op in plan.ops:
            if op[2] in G.ARGS:
                G.decode(op)


def test_odd_geometry_runs_the_generic_resize(graphs):
    """100x172: the recover decoder's 4x6 -> 7x11 -> 13x22 -> 25x43 resize-concats take the generic (non-x2) kernel and transpose."""
    kinds = collections.Counter()
    for name, plan in graphs['odd'].items():
        for op in plan.ops:
            if op[2].startswith('cis_resize_concat_bf16'):
                a = G.decode(op)
                kinds[(name, G.Glue._rc_kind(a['H'], a['W'], a['OH'], a['OW']))] += 1
    assert kinds[('fwd', 'generic')] == 6 and kinds[('bwd_R', 'generic')] == 6 and kinds[('bwd_G', 'generic')] == 6, kinds
