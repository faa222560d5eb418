"""GPU parity of the halo conv kernel with two MMA warpgroups per CTA (CisConv.nwg = 2) against the fp32 reference of
tests/convref.py, and bit-identity with the one-warpgroup kernel: both run the same wgmma in the same K order for every output
element, only the CTA that owns the element changes."""
import pytest

from convref import run_conv_case
from unsupervised_detection_b200 import engine
from unsupervised_detection_b200._lib import ACT_ELU, ACT_LEAKY

pytestmark = pytest.mark.gpu

CASES = [
    # BN = 128, one tile per warpgroup, ragged last CTA row (70 = 2 x 32 + 6)
    dict(N=2, H=70, W=44, cins=[128], cout=128, k=3, act=ACT_ELU, bn=True),
    # BN = 64 (MT = 2 per warpgroup is forced below)
    dict(N=2, H=96, W=64, cins=[128], cout=64, k=3, act=ACT_LEAKY),
    # dilated layer (dilation phases, taller TMA box in dilated pixel space)
    dict(N=1, H=50, W=36, cins=[128], cout=128, k=3, dil=2, act=ACT_ELU, bn=True),
    # stride-2 layer: its data gradient is one grouped launch of the 4 output parities (CisConv.nsub = 4, BN = 128)
    dict(N=2, H=64, W=48, cins=[128], cout=64, k=3, stride=2, act=ACT_ELU),
    # concatenated sources with a batch-broadcast (n_mod) last source, even kernel (asymmetric halo)
    dict(N=6, H=40, W=24, cins=[64, 64, 64], cout=64, k=4, act=ACT_LEAKY, n_mod_last=2),
    # a first source that is not a multiple of 64 channels: the cp.async halo path instead of the TMA one
    dict(N=4, H=48, W=40, cins=[40, 64], cout=128, k=3, backward=False),
]
IDS = ['bn128', 'bn64_mt2', 'dil2', 's2_grouped_dgrad', 'concat_nmod', 'cp_async_halo']


def _tol(ref):
    return 2 ** -7 * ref + 1e-3


def _run(monkeypatch, case, nwg_mode, mt64=False):
    """run_conv_case with engine.HALO_NWG = nwg_mode; returns (errors, list of the nwg values the planner chose)."""
    chosen = []
    orig = engine.halo_nwg

    def rec(d, MT, *a):
        if mt64 and d.BN == 64 and d.MT == 1:
            d.MT = MT = 2
        v = orig(d, MT, *a)
        chosen.append(v)
        return v

    with monkeypatch.context() as m:
        m.setattr(engine, 'HALO_NWG', nwg_mode)
        m.setattr(engine, 'halo_nwg', rec)
        r = run_conv_case(**case)
    return r, chosen


def _check(r):
    assert r['fwd_err'] <= _tol(r['fwd_ref']), r
    if 'dx_err' in r:
        assert r['dx_err'] <= _tol(r['dx_ref']), r
        assert r['dw_err'] <= 2 ** -7 * r['dw_ref'] + 1e-3, r


def _same(r1, r2):
    for k in ('fwd_err', 'dx_err', 'dw_err'):
        if k in r1:
            assert r1[k] == r2[k], (k, r1, r2)


@pytest.mark.parametrize('case', CASES, ids=IDS)
def test_two_warpgroups_match_reference_and_one_warpgroup(monkeypatch, case):
    mt64 = case is CASES[1]
    r1, c1 = _run(monkeypatch, case, 1, mt64)
    r2, c2 = _run(monkeypatch, case, 3, mt64)
    assert set(c1) == {1} and 2 in c2, (c1, c2)
    _check(r2)
    _same(r1, r2)


@pytest.mark.parametrize('cluster', [False, True], ids=['two_launch', 'cluster'])
@pytest.mark.parametrize('case', [CASES[0], CASES[1], CASES[4]], ids=['bn128', 'bn64_mt2', 'concat_nmod'])
def test_two_warpgroups_split_k(monkeypatch, case, cluster):
    """Split-K forced onto the taller CTAs: the two-launch form (one scratch slice per 16x8 tile of the CTA and split, finish
    kernel) and the thread-block-cluster form (DSMEM reduction of all 2*MT tiles).  The split factor follows the CTA count, so
    the summation order may differ from the one-warpgroup plan: checked against the reference."""
    splits = []
    orig_splitk = engine.setup_splitk

    def rec_splitk(d, *a):
        orig_splitk(d, *a)
        splits.append((d.nwg, d.splits))

    monkeypatch.setattr(engine, 'SPLITK', 2)
    monkeypatch.setattr(engine, 'SPLITK_NCTA', 10 ** 6)
    monkeypatch.setattr(engine, 'SPLITK_MIN_UNITS', 0)
    monkeypatch.setattr(engine, 'SPLITK_CLUSTER', cluster)
    monkeypatch.setattr(engine, 'setup_splitk', rec_splitk)
    r, chosen = _run(monkeypatch, case, 3, case is CASES[1])
    assert any(n == 2 and s > 1 for n, s in splits), splits
    _check(r)
