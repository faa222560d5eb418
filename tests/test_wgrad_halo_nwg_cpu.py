"""Planner side of the halo weight-gradient tiling (CisWgrad.nh / nwg, engine.wgrad_halo_tiling), on the step graph BUILT on CPU
tensors at the benchmark size (256x448, batch 4): every tma = 2 descriptor keeps a warpgroup's accumulator in 128 registers per thread,
fits shared memory as launch_wgrad_halo_t sizes it, and gives every split a pixel block; and the MMA work the plan issues is close to
the useful work (real input and output channels)."""
import pytest

from unsupervised_detection_b200 import engine
from unsupervised_detection_b200.step_graph import CISGraph

SMEM = 227 * 1024


def _wgrad_halo(g):
    for plan, w in ((g.bwd['G'], 3), (g.bwd['R'], 1)):       # per step: 1 recover step for 3 generator steps
        for fn, a, name, fl, lane in plan.ops:
            if name == 'cis_conv_wgrad' and a[0]._obj.tma == 2:
                yield a[0]._obj, w / 4.0


def _geometry(d):
    chunks = sum(d.src[i].chunks for i in range(d.nsrc))
    taps = [(d.dh[t], d.dw[t]) for t in range(d.ntaps)]
    wh = 8 + max(b for _, b in taps) - min(b for _, b in taps)
    hh = 8 + max(a for a, _ in taps) - min(a for a, _ in taps)
    nblk = d.N * (-(-d.OH // 8)) * (-(-d.OW // 8))
    return chunks * 8, -(-chunks // 8), wh, hh, nblk


def _pairs_per_cta(d):
    """Tap pairs each CTA along grid.z issues per warpgroup (launch_wgrad_halo_t / wgrad_halo_wg_pairs)."""
    nh, nwg = d.nh or 64, max(d.nwg, 1)
    p, npairs = 128 // nh, (d.ntaps + 1) // 2
    if nwg == 2 and d.Cout > 64:
        return [[min(p, npairs - q0)] * 2 for q0 in range(0, npairs, p)]
    out = []
    for q0 in range(0, npairs, nwg * p):
        cnt = min(nwg * p, npairs - q0)
        h = -(-cnt // 2) if nwg == 2 else cnt
        out += [[h, cnt - h] if nwg == 2 else [h]] * (2 if d.Cout > 64 else 1)
    return out


def _work(g):
    useful = issued = 0.0
    for d, w in _wgrad_halo(g):
        cin, nch64, _, _, nblk = _geometry(d)
        useful += w * 2.0 * d.N * d.OH * d.OW * d.ntaps * cin * d.Cout
        pairs = sum(sum(c) for c in _pairs_per_cta(d))
        issued += w * nblk * nch64 * pairs * 2.0 * 128 * (d.nh or 64) * 64
    return useful, issued


@pytest.fixture(scope='module')
def bench_graph():
    return CISGraph(256, 448, 4, device='cpu')


def test_tma2_descriptors_fit_registers_smem_and_splits(bench_graph):
    n = 0
    for d, _ in _wgrad_halo(bench_graph):
        n += 1
        nh, nwg = d.nh or 64, max(d.nwg, 1)
        assert nh in (16, 32, 64) and nwg in (1, 2)
        assert nh >= min(64, -(-d.Cout // 16) * 16) and (d.Cout <= 64 or nh == 64)
        for per_wg in _pairs_per_cta(d):
            assert len(per_wg) == nwg and max(per_wg) * nh <= engine.MAX_ACC_COLS
        _, _, wh, hh, nblk = _geometry(d)
        stage = -(-(wh * hh * 128) // 1024) * 1024 + (2 if nwg == 2 and d.Cout > 64 else 1) * 64 * 2 * nh
        s = min(6, (200 * 1024) // stage)
        assert s >= 2
        assert max(s * stage, nwg * engine.MAX_ACC_COLS * 512) + 1024 <= SMEM     # the accumulators overlay the stage ring
        per = -(-nblk // d.splits)
        assert (d.splits - 1) * per < nblk                                         # every split owns a pixel block
        assert d.splits * d.Cout * d.K_pad * 4 <= max(engine.WGRAD_MAX_SLICE_MB * 1e6, d.Cout * d.K_pad * 4)
    assert n > 0


def test_issued_mma_work_close_to_useful(bench_graph, monkeypatch):
    useful, issued = _work(bench_graph)
    assert issued / useful <= 1.35, (useful / 1e9, issued / 1e9)
    monkeypatch.setattr(engine, 'WGRAD_HALO_NWG', 1)
    u1, i1 = _work(CISGraph(256, 448, 4, device='cpu'))
    assert u1 == useful and i1 / u1 >= 2.0, (u1 / 1e9, i1 / 1e9)


def test_wgrad_halo_nwg_1_keeps_the_n64_one_warpgroup_tiling(monkeypatch):
    monkeypatch.setattr(engine, 'WGRAD_HALO_NWG', 1)
    g = CISGraph(128, 224, 4, device='cpu')
    ds = [d for d, _ in _wgrad_halo(g)]
    assert ds and all((d.nh, d.nwg) == (64, 1) for d in ds)


@pytest.mark.parametrize('ntaps,cout,expect', [
    (9, 2, (16, 1, 1)), (9, 16, (16, 1, 1)), (9, 32, (32, 2, 1)), (9, 64, (64, 2, 2)), (9, 128, (64, 2, 3)),
    (16, 16, (16, 1, 1)), (16, 128, (64, 2, 4)), (25, 2, (16, 2, 1)), (25, 32, (32, 2, 2))])
def test_wgrad_halo_tiling(ntaps, cout, expect):
    assert engine.wgrad_halo_tiling(ntaps, cout) == expect
