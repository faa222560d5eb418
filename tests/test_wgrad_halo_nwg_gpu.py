"""GPU parity of the halo weight-gradient kernel's tilings (CisWgrad.nh / nwg, engine.wgrad_halo_tiling): narrow MMA N (16 / 32 output
channels, 32B / 64B-swizzled gradient tiles), two MMA warpgroups splitting a CTA's tap pairs (Cout <= 64) or taking the two Cout
halves (Cout > 64), odd pair counts and a warpgroup without pairs.  Checked against the fp32 reference of tests/convref.py with the
tolerance of test_conv_engine_halo_wgrad, and against the one-warpgroup N = 64 tiling (CIS_WGRAD_HALO_NWG=1) at equal splits."""
import pytest
import torch

from convref import run_conv_case
from unsupervised_detection_b200 import engine

pytestmark = pytest.mark.gpu

CASES = [
    # 3x3 (5 pairs): every nh, one and two warpgroups, input channels whose last 64-channel chunk is partial
    dict(N=2, H=40, W=48, cins=[56], cout=2, k=3),                      # nh 16, nwg 1
    dict(N=2, H=40, W=48, cins=[104], cout=16, k=3),                    # nh 16, nwg 1
    dict(N=2, H=40, W=48, cins=[200], cout=32, k=3),                    # nh 32, nwg 2: 3 + 2 pairs
    dict(N=2, H=33, W=50, cins=[104], cout=64, k=3),                    # nh 64, nwg 2: 2 + 2 pairs, then 1 + 0
    dict(N=2, H=24, W=40, cins=[200], cout=128, k=3),                   # nh 64, nwg 2: the two Cout halves
    # 4x4 (16 taps, 8 pairs)
    dict(N=2, H=40, W=48, cins=[104], cout=16, k=4),                    # nh 16, nwg 1: 8 pairs in one warpgroup
    dict(N=2, H=32, W=40, cins=[56], cout=32, k=4),                     # nh 32, nwg 2: 4 + 4 pairs
    dict(N=2, H=24, W=32, cins=[128], cout=128, k=4),                   # nh 64, nwg 2: halves, 4 pair groups
    # 5x5 (25 taps, 13 pairs, odd last pair)
    dict(N=2, H=40, W=48, cins=[56], cout=2, k=5),                      # nh 16, nwg 2: 7 + 6 pairs
    dict(N=2, H=32, W=40, cins=[104], cout=32, k=5),                    # nh 32, nwg 2: 4 + 4 pairs, 3 + 2 pairs
    # concatenated sources, the last one broadcast over the batch (n_mod)
    dict(N=4, H=24, W=32, cins=[64, 64, 16], cout=32, k=3, n_mod_last=2),
    dict(N=4, H=24, W=32, cins=[64, 40], cout=128, k=3, n_mod_last=2),
]


def _ids(c):
    return 'k%d_c%s_o%d_%dx%dx%d' % (c['k'], '+'.join(map(str, c['cins'])), c['cout'], c['N'], c['H'], c['W'])


_ENGINE = (engine.ParamStore, engine.wgrad_halo_tiling, engine.ConvLayer)


def _run(monkeypatch, case, nwg_env, ctas_per_sm):
    """One forward + backward of the case on the halo wgrad path; returns (errors, dw, tilings planned, wgrad splits)."""
    stores, tilings, layers = [], [], []
    real_store, real_tiling, real_layer = _ENGINE

    class Store(real_store):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            stores.append(self)

    class Layer(real_layer):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            layers.append(self)

    def tiling(ntaps, cout):
        t = real_tiling(ntaps, cout)
        tilings.append(t)
        return t

    monkeypatch.setattr(engine, 'WGRAD_HALO', True)
    monkeypatch.setattr(engine, 'WGRAD_HALO_NWG', nwg_env)
    monkeypatch.setattr(engine, 'WGRAD_CTAS_PER_SM', ctas_per_sm)
    monkeypatch.setattr(engine, 'ParamStore', Store)
    monkeypatch.setattr(engine, 'ConvLayer', Layer)
    monkeypatch.setattr(engine, 'wgrad_halo_tiling', tiling)
    r = run_conv_case(**case)
    dw = stores[-1].view('L/kernel', 'grad').clone()
    return r, dw, tilings, dict(layers[-1].wg_splits)


@pytest.mark.parametrize('case', CASES, ids=_ids)
def test_wgrad_halo_tiling_matches_reference(monkeypatch, case):
    r, _, tilings, splits = _run(monkeypatch, case, 2, engine.WGRAD_CTAS_PER_SM)
    assert tilings, 'the layer did not take the halo wgrad kernel'
    nh, nwg, _ = tilings[-1]
    assert nh == min(64, -(-case['cout'] // 16) * 16)
    assert r['dw_err'] <= 2 ** -7 * r['dw_ref'] + 1e-3, (r, tilings[-1], splits)
    assert r['db_err'] <= 2 ** -7 * r['db_ref'] + 1e-3, r


@pytest.mark.parametrize('ctas_per_sm', [0, 10 ** 4])
@pytest.mark.parametrize('case', [CASES[i] for i in (1, 2, 3, 4, 8, 10)], ids=_ids)
def test_wgrad_halo_tiling_matches_one_warpgroup_n64(monkeypatch, case, ctas_per_sm):
    """Same splits (one, or as many as the pixel blocks allow) under both tilings: only the MMA N and the CTA a tap pair runs in
    differ, so the weight gradients agree to fp32 summation-order level (each split sums its pixel blocks in the same order)."""
    r1, dw1, t1, s1 = _run(monkeypatch, case, 1, ctas_per_sm)
    r2, dw2, t2, s2 = _run(monkeypatch, case, 2, ctas_per_sm)
    assert t1[-1][:2] == (64, 1) and s1 == s2, (t1, t2, s1, s2)
    scale = float(dw1.abs().max())
    assert float((dw2 - dw1).abs().max()) <= 1e-5 * scale, (s1, t2)
    assert r2['dw_err'] <= 2 ** -7 * r2['dw_ref'] + 1e-3, r2


def test_wgrad_halo_tiling_is_deterministic(monkeypatch):
    case = CASES[8]
    _, dwa, _, _ = _run(monkeypatch, case, 2, engine.WGRAD_CTAS_PER_SM)
    _, dwb, _, _ = _run(monkeypatch, case, 2, engine.WGRAD_CTAS_PER_SM)
    assert torch.equal(dwa, dwb)
