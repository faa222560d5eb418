"""Planner side of the two-MMA-warpgroup halo kernel (CisConv.nwg), on the step graph BUILT on CPU tensors at the benchmark size
(256x448, batch 4, PWC-Net at 384x640): which launches take two warpgroups, and that every such descriptor fits the launcher's
shared-memory and utilisation bounds computed with the real CTA height of 16 * nwg * MT rows."""
import pytest

from unsupervised_detection_b200 import engine
from unsupervised_detection_b200.step_graph import CISGraph


def _halo_convs(g):
    for plan in (g.fwd, g.bwd['G'], g.bwd['R']):
        for fn, a, name, fl, lane in plan.ops:
            if name == 'cis_conv_igemm' and a[0]._obj.halo:
                yield a[0]._obj


@pytest.fixture(scope='module')
def bench_graph():
    return CISGraph(256, 448, 4, device='cpu')


def test_pwc_96x160_bn128_layers_take_two_warpgroups(bench_graph):
    pwc = [d for d in _halo_convs(bench_graph) if d.BN == 128 and d.dil == 1 and d.N == 4 and (d.OH, d.OW) == (96, 160)]
    assert len(pwc) >= 4
    assert all(d.nwg == 2 and d.MT == 1 for d in pwc), [(d.MT, d.nwg) for d in pwc]


def test_two_warpgroup_descriptors_fit_the_launcher(bench_graph):
    n = 0
    for d in _halo_convs(bench_graph):
        assert d.nwg in (0, 1, 2)
        if d.nwg != 2:
            continue
        n += 1
        mtc = 2 * d.MT
        assert d.BN >= 64 and d.MT * d.BN <= engine.MAX_ACC_COLS          # per warpgroup
        hp = (8 + d.ex) * (16 * mtc + d.ey)
        nhs = 2
        assert nhs * ((hp * 128 + 1023) // 1024 * 1024) + hp * 4 + 1024 + d.BN * 128 <= 227 * 1024   # a weight stage beside the halo
        assert mtc * 128 * d.BN * 4 + 1024 <= 226 * 1024                   # the fp32 tiles of both warpgroups overlay the operands
        hp0, wp0 = -(-d.OH // d.dil), -(-d.OW // d.dil)
        util = hp0 * wp0 / float((-(-hp0 // (16 * mtc))) * 16 * mtc * (-(-wp0 // 8)) * 8)
        assert util >= (engine.HALO_MIN_UTIL if d.dil == 1 else 0.5)
    assert n > 0


def test_halo_nwg_1_keeps_one_warpgroup(monkeypatch):
    monkeypatch.setattr(engine, 'HALO_NWG', 1)
    g = CISGraph(128, 224, 4, device='cpu')
    assert all(d.nwg <= 1 for d in _halo_convs(g))
