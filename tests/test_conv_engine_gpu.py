"""GPU parity of the wgmma implicit-GEMM conv engine (forward, data gradient, weight gradient) against a plain torch
fp32 reference of the same op on the same bf16-rounded operands.  Tolerances: the product accumulates in fp32 from bf16
operands exactly like the reference's inputs, so only summation order and the final bf16 rounding of stored activations
differ: |err| <= 2^-8 * |ref|_max + small absolute slack."""
import os

import pytest
import torch

from convref import run_conv_case
from unsupervised_detection_b200._lib import ACT_NONE, ACT_ELU, ACT_LEAKY

pytestmark = pytest.mark.gpu

CASES = [
    # N, H, W, cins, cout, k, stride, dil, act, bn, post_add
    dict(N=2, H=16, W=24, cins=[64], cout=64, k=3),
    dict(N=2, H=16, W=24, cins=[128], cout=128, k=3, act=ACT_ELU, bn=True),
    dict(N=1, H=32, W=40, cins=[5], cout=32, k=5, act=ACT_ELU, bn=True),
    dict(N=2, H=16, W=28, cins=[32], cout=64, k=3, stride=2, act=ACT_ELU, bn=True),
    dict(N=1, H=24, W=24, cins=[128], cout=128, k=3, dil=4, act=ACT_ELU, bn=True, post_add=True),
    dict(N=1, H=17, W=23, cins=[3], cout=16, k=7, stride=2, act=ACT_LEAKY),
    dict(N=3, H=8, W=14, cins=[128, 128, 128, 2], cout=128, k=4, act=ACT_LEAKY, n_mod_last=0),
    dict(N=3, H=8, W=14, cins=[128, 128, 2, 128], cout=2, k=3),
    dict(N=6, H=9, W=7, cins=[64, 64, 64], cout=64, k=4, act=ACT_LEAKY, n_mod_last=2),
    dict(N=1, H=12, W=20, cins=[16], cout=32, k=5, stride=2, act=ACT_LEAKY),
    dict(N=2, H=6, W=10, cins=[196], cout=196, k=3, act=ACT_LEAKY, alpha=0.1, backward=False),
    dict(N=1, H=20, W=20, cins=[16], cout=2, k=3),
    # larger maps: exercise the halo-resident kernel with several stacked M tiles, ragged tiles and dilation phases
    dict(N=2, H=70, W=44, cins=[128], cout=128, k=3, act=ACT_ELU, bn=True),
    dict(N=4, H=96, W=160, cins=[64, 40], cout=128, k=3, act=ACT_LEAKY, alpha=0.1, backward=False),
    dict(N=1, H=50, W=36, cins=[128], cout=128, k=3, dil=2, act=ACT_ELU, bn=True),
    dict(N=1, H=64, W=112, cins=[128], cout=96, k=3, dil=8, act=ACT_LEAKY, backward=False),
    dict(N=3, H=40, W=56, cins=[16, 16, 16, 2], cout=2, k=5),
    dict(N=3, H=33, W=57, cins=[32, 32, 32, 2], cout=16, k=4, act=ACT_LEAKY),
    dict(N=2, H=40, W=48, cins=[5], cout=32, k=5, act=ACT_ELU, bn=True),
]


@pytest.mark.parametrize('case', CASES, ids=lambda c: 'k%d_s%d_d%d_c%s_o%d' % (c['k'], c.get('stride', 1), c.get('dil', 1), '+'.join(map(str, c['cins'])), c['cout']))
def test_conv_engine(case):
    r = run_conv_case(**case)
    tol = lambda ref: 2 ** -7 * ref + 1e-3
    assert r['fwd_err'] <= tol(r['fwd_ref']), r
    if 'dx_err' in r:
        assert r['dx_err'] <= tol(r['dx_ref']), r
        assert r['dw_err'] <= 2 ** -7 * r['dw_ref'] + 1e-3, r   # g*act' is stored in bf16 before the wgrad GEMM
        assert r['db_err'] <= 2 ** -7 * r['db_ref'] + 1e-3, r
    if 'dgamma_err' in r:
        assert r['dgamma_err'] <= 2 ** -6 * r['dgamma_ref'] + 1e-2, r
        assert r['dbeta_err'] <= 2 ** -6 * r['dbeta_ref'] + 1e-2, r


MODE_CASES = [CASES[0], CASES[1], CASES[4], CASES[6], CASES[11], CASES[12], CASES[14], CASES[17]]


@pytest.mark.parametrize('case', MODE_CASES, ids=lambda c: 'k%d_d%d_c%s_o%d' % (c['k'], c.get('dil', 1), '+'.join(map(str, c['cins'])), c['cout']))
def test_conv_engine_persistent_kernel_everywhere(case):
    """Force the persistent warp-specialised halo kernel for every eligible launch (default: thin layers only)."""
    from unsupervised_detection_b200 import _lib
    _lib.load().cis_set_persist_mode(2)
    try:
        r = run_conv_case(**case)
    finally:
        _lib.load().cis_set_persist_mode(-1)
    tol = lambda ref: 2 ** -7 * ref + 1e-3
    assert r['fwd_err'] <= tol(r['fwd_ref']), r
    if 'dx_err' in r:
        assert r['dx_err'] <= tol(r['dx_ref']), r
        assert r['dw_err'] <= 2 ** -7 * r['dw_ref'] + 1e-3, r


@pytest.mark.parametrize('case', MODE_CASES, ids=lambda c: 'k%d_d%d_c%s_o%d' % (c['k'], c.get('dil', 1), '+'.join(map(str, c['cins'])), c['cout']))
def test_conv_engine_split_k(case):
    """Split-K (private fp32 slices + the parallel finish kernel, engine.SPLITK = 2, the default for low-resolution launches) forced
    onto every case: same tolerance as the unsplit kernels, and bit-reproducible run to run (fixed summation order)."""
    from unsupervised_detection_b200 import engine
    old = (engine.SPLITK, engine.SPLITK_NCTA, engine.SPLITK_MIN_UNITS)
    engine.SPLITK, engine.SPLITK_NCTA, engine.SPLITK_MIN_UNITS = 2, 10 ** 6, 0
    try:
        r = run_conv_case(**case)
        r2 = run_conv_case(**case)
    finally:
        engine.SPLITK, engine.SPLITK_NCTA, engine.SPLITK_MIN_UNITS = old
    tol = lambda ref: 2 ** -7 * ref + 1e-3
    assert r['fwd_err'] <= tol(r['fwd_ref']), r
    assert r['fwd_err'] == r2['fwd_err']
    if 'dx_err' in r:
        assert r['dx_err'] <= tol(r['dx_ref']), r
        assert r['dx_err'] == r2['dx_err']


WS_CASES = [CASES[2], CASES[11], CASES[16], CASES[17], CASES[18], CASES[0],
            dict(N=2, H=64, W=96, cins=[5], cout=32, k=5, act=ACT_ELU, bn=True, backward=False),
            dict(N=3, H=48, W=80, cins=[16, 16, 16, 2], cout=2, k=5, backward=False)]


@pytest.mark.parametrize('case', WS_CASES, ids=lambda c: 'k%d_c%s_o%d_%dx%d' % (c['k'], '+'.join(map(str, c['cins'])), c['cout'], c['H'], c['W']))
def test_conv_engine_weight_stationary_persistent(case):
    """Persist mode 3: thin layers whose whole weight set fits in shared memory keep it resident across the tiles of a CTA."""
    from unsupervised_detection_b200 import _lib
    r0 = run_conv_case(**case)
    _lib.load().cis_set_persist_mode(3)
    try:
        r = run_conv_case(**case)
    finally:
        _lib.load().cis_set_persist_mode(-1)
    tol = lambda ref: 2 ** -7 * ref + 1e-3
    assert r['fwd_err'] <= tol(r['fwd_ref']), r
    assert r['fwd_err'] == r0['fwd_err']          # same MMAs in the same order: bit-identical to the default kernels
    if 'dx_err' in r:
        assert r['dx_err'] <= tol(r['dx_ref']), r


WGH_CASES = [CASES[0], CASES[1], CASES[2], CASES[4], CASES[6], CASES[7], CASES[11], CASES[12], CASES[14], CASES[16], CASES[17], CASES[18]]


@pytest.mark.parametrize('case', WGH_CASES, ids=lambda c: 'k%d_d%d_c%s_o%d' % (c['k'], c.get('dil', 1), '+'.join(map(str, c['cins'])), c['cout']))
def test_conv_engine_halo_wgrad(case, monkeypatch):
    """CisWgrad.tma = 2 (engine.WGRAD_HALO): swapped, halo-resident weight gradient; same tolerance as the default kernels."""
    from unsupervised_detection_b200 import engine
    monkeypatch.setattr(engine, 'WGRAD_HALO', True)     # restored afterwards: later tests plan with the configured default
    r = run_conv_case(**case)
    assert r['dw_err'] <= 2 ** -7 * r['dw_ref'] + 1e-3, r
    assert r['db_err'] <= 2 ** -7 * r['db_ref'] + 1e-3, r
    if 'dgamma_err' in r:
        assert r['dgamma_err'] <= 2 ** -6 * r['dgamma_ref'] + 1e-2, r
        assert r['dbeta_err'] <= 2 ** -6 * r['dbeta_ref'] + 1e-2, r


NARROW_CASES = [CASES[1], CASES[6], CASES[10], CASES[12], CASES[13], CASES[4]]


@pytest.mark.parametrize('cap', [32, 64])
@pytest.mark.parametrize('case', NARROW_CASES, ids=lambda c: 'k%d_d%d_c%s_o%d' % (c['k'], c.get('dil', 1), '+'.join(map(str, c['cins'])), c['cout']))
def test_conv_engine_narrow_n_tiles(case, cap):
    """ConvLayer(bn_cap=...): Cout > cap is covered by several BN = cap n-tiles instead of BN = 128 (more CTAs on tiny maps)."""
    r = run_conv_case(bn_cap=cap, **case)
    tol = lambda ref: 2 ** -7 * ref + 1e-3
    assert r['fwd_err'] <= tol(r['fwd_ref']), r
    if 'dx_err' in r:
        assert r['dx_err'] <= tol(r['dx_ref']), r
        assert r['dw_err'] <= 2 ** -7 * r['dw_ref'] + 1e-3, r


S2_CASES = [c for c in CASES if c.get('stride', 1) == 2]


@pytest.mark.parametrize('case', S2_CASES, ids=lambda c: 'k%d_c%s_o%d' % (c['k'], '+'.join(map(str, c['cins'])), c['cout']))
def test_conv_engine_stride2_on_the_halo_kernel(case):
    """engine.S2_HALO (off by default): stride-2 forward convs as four space-to-depth phase halos (CisConv.nph = 4, TMA phase maps)."""
    from unsupervised_detection_b200 import engine
    assert S2_CASES
    engine.S2_HALO = True
    try:
        r = run_conv_case(**case)
    finally:
        engine.S2_HALO = False
    tol = lambda ref: 2 ** -7 * ref + 1e-3
    assert r['fwd_err'] <= tol(r['fwd_ref']), r
    if 'dx_err' in r:
        assert r['dx_err'] <= tol(r['dx_ref']), r
        assert r['dw_err'] <= 2 ** -7 * r['dw_ref'] + 1e-3, r


@pytest.mark.parametrize('case', MODE_CASES, ids=lambda c: 'k%d_d%d_c%s_o%d' % (c['k'], c.get('dil', 1), '+'.join(map(str, c['cins'])), c['cout']))
def test_conv_engine_split_k_cluster(case):
    """engine.SPLITK_CLUSTER: the splits of a tile form a thread-block cluster (<= 8 CTAs along grid.z) and reduce their partial
    accumulators through distributed shared memory inside the conv kernel -- same tolerance, bit-reproducible, no finish launch."""
    from unsupervised_detection_b200 import engine
    old = (engine.SPLITK, engine.SPLITK_NCTA, engine.SPLITK_MIN_UNITS, engine.SPLITK_CLUSTER)
    engine.SPLITK, engine.SPLITK_NCTA, engine.SPLITK_MIN_UNITS, engine.SPLITK_CLUSTER = 2, 10 ** 6, 0, True
    try:
        r = run_conv_case(**case)
        r2 = run_conv_case(**case)
    finally:
        engine.SPLITK, engine.SPLITK_NCTA, engine.SPLITK_MIN_UNITS, engine.SPLITK_CLUSTER = old
    tol = lambda ref: 2 ** -7 * ref + 1e-3
    assert r['fwd_err'] <= tol(r['fwd_ref']), r
    assert r['fwd_err'] == r2['fwd_err']
    if 'dx_err' in r:
        assert r['dx_err'] <= tol(r['dx_ref']), r
        assert r['dx_err'] == r2['dx_err']
