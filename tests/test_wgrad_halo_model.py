"""Index-level model of the halo-resident wgrad kernel (csrc/conv_igemm.cu: conv_wgrad_halo_kernel, CisWgrad.tma = 2).

What CAN be checked without a GPU is its addressing scheme: this test replays, in numpy, exactly
the data movement the kernel programs -- the zero-filled TMA halo box, the tap origins `s_off`, the per-K-step descriptor start
(two halo rows per 16 pixels), the LBO hop from tap 2q to tap 2q+1 inside one M = 128 operand, the accumulator column ranges and
the epilogue's (tap, chunk, channel) -> packed column map -- and compares the result with a direct weight-gradient sum.
What it cannot check is the hardware's treatment of those descriptors (tests/test_conv_engine_gpu.py runs the kernel)."""
import numpy as np
import pytest

from unsupervised_detection_b200.engine import wgrad_halo_fits, ru


def model_wgrad_halo(x, g, taps, cout):
    N, H, W, C = x.shape
    _, OH, OW, _ = g.shape
    ntaps = len(taps)
    nch64 = -(-C // 64)
    hoy, hox = min(a for a, _ in taps), min(b for _, b in taps)
    Wh, Hh = 8 + max(b for _, b in taps) - hox, 8 + max(a for a, _ in taps) - hoy
    s_off = [(a - hoy) * Wh + (b - hox) for a, b in taps] + [0]
    npair = (ntaps + 1) // 2
    Nh = 64 if cout > 64 else ru(cout, 16)
    nhalf = 2 if cout > 64 else 1
    K_pad = ru(ntaps * nch64 * 64, 128)
    dwp = np.zeros((cout, K_pad), np.float64)
    tiles_y, tiles_x = -(-OH // 8), -(-OW // 8)
    for c64 in range(nch64):
        for half in range(nhalf):
            acc = np.zeros((npair, 128, Nh), np.float64)                      # accumulator: pair q -> columns [q*Nh, (q+1)*Nh)
            for n in range(N):
                for ty in range(tiles_y):
                    for tx in range(tiles_x):
                        halo = np.zeros((Hh * Wh + 2 * Wh + 16, 64), np.float64)   # flat pixel rows (+ slack for the phantom tap)
                        for hy in range(Hh):
                            for hx in range(Wh):
                                y, xx = ty * 8 + hoy + hy, tx * 8 + hox + hx
                                if 0 <= y < H and 0 <= xx < W:
                                    ch = x[n, y, xx, c64 * 64:(c64 + 1) * 64]
                                    halo[hy * Wh + hx, :len(ch)] = ch               # channels past C: TMA zero fill
                        gt = np.zeros((64, 64), np.float64)
                        for py in range(8):
                            for px in range(8):
                                y, xx = ty * 8 + py, tx * 8 + px
                                if y < OH and xx < OW:
                                    ch = g[n, y, xx, half * 64:(half + 1) * 64]
                                    gt[py * 8 + px, :len(ch)] = ch
                        for q in range(npair):
                            o0, o1 = s_off[2 * q], s_off[2 * q + 1]
                            lbo = o1 - o0 if o1 > o0 else 1
                            for k in range(4):
                                start = o0 + 2 * k * Wh
                                for j in range(16):
                                    row = start + (j // 8) * Wh + (j % 8)           # SBO = one halo row between 8-pixel groups
                                    a = np.concatenate([halo[row], halo[row + lbo]])   # MN atoms: tap 2q, tap 2q+1
                                    acc[q] += np.outer(a, gt[16 * k + j, :Nh])
            for q in range(npair):
                for m in range(128):
                    t = 2 * q + m // 64
                    if t >= ntaps:
                        continue
                    kcol = (t * nch64 + c64) * 64 + m % 64
                    for e in range(Nh):
                        co = half * 64 + e
                        if co < cout:
                            dwp[co, kcol] += acc[q, m, e]
    return dwp, nch64


def direct_wgrad(x, g, taps, cout):
    N, H, W, C = x.shape
    _, OH, OW, _ = g.shape
    dw = np.zeros((len(taps), C, cout), np.float64)
    xp = np.pad(x, ((0, 0), (64, 64), (64, 64), (0, 0)))
    for t, (a, b) in enumerate(taps):
        xs = xp[:, 64 + a:64 + a + OH, 64 + b:64 + b + OW, :]
        dw[t] = np.einsum('nhwc,nhwo->co', xs, g)
    return dw


CASES = [
    dict(N=1, H=11, W=13, C=5, cout=3, taps=[(a, b) for a in (-1, 0, 1) for b in (-1, 0, 1)]),                 # 3x3 SAME, ragged tiles
    dict(N=2, H=8, W=16, C=70, cout=20, taps=[(a, b) for a in (-2, -1, 0, 1, 2) for b in (-2, -1, 0, 1, 2)]),   # 5x5, two 64-ch chunks
    dict(N=1, H=9, W=9, C=8, cout=70, taps=[(a, b) for a in (-1, 0, 1, 2) for b in (-1, 0, 1, 2)]),             # 4x4 (asymmetric pad), two Cout halves
    dict(N=1, H=12, W=10, C=6, cout=2, taps=[(a, b) for a in (-2, 0, 2) for b in (-2, 0, 2)]),                  # 3x3 dilation 2
]


@pytest.mark.parametrize('case', CASES, ids=lambda c: '%dtaps_C%d_o%d' % (len(c['taps']), c['C'], c['cout']))
def test_halo_wgrad_addressing_model(case):
    rng = np.random.RandomState(len(case['taps']) + case['C'])
    x = rng.randint(-3, 4, (case['N'], case['H'], case['W'], case['C'])).astype(np.float64)
    g = rng.randint(-3, 4, (case['N'], case['H'], case['W'], case['cout'])).astype(np.float64)
    assert wgrad_halo_fits(case['taps'], case['cout'], 1)
    dwp, nch64 = model_wgrad_halo(x, g, case['taps'], case['cout'])
    ref = direct_wgrad(x, g, case['taps'], case['cout'])
    for t in range(len(case['taps'])):
        for c in range(case['C']):
            kcol = (t * nch64 + c // 64) * 64 + c % 64
            assert np.array_equal(dwp[:, kcol], ref[t, c]), (t, c)
    # columns that belong to no (tap, channel) stay zero (they are dropped by cis_unpack_wgrad's kmap = -1)
    used = {(t * nch64 + c // 64) * 64 + c % 64 for t in range(len(case['taps'])) for c in range(case['C'])}
    rest = [k for k in range(dwp.shape[1]) if k not in used]
    assert not dwp[:, rest].any()


def test_halo_wgrad_eligibility_rules():
    t3 = [(a, b) for a in (-1, 0, 1) for b in (-1, 0, 1)]
    assert wgrad_halo_fits(t3, 128, 1) and not wgrad_halo_fits(t3, 128, 2)
    assert not wgrad_halo_fits(t3[::-1], 16, 1)                                   # pairs need increasing row-major origins
    t5 = [(a, b) for a in range(-2, 3) for b in range(-2, 3)]
    assert wgrad_halo_fits(t5, 32, 1) and not wgrad_halo_fits(t5, 128, 1)         # 13 pairs x 64 columns exceed the 512 the planner allows
    assert not wgrad_halo_fits([(a * 16, b * 16) for a in (-1, 0, 1) for b in (-1, 0, 1)], 128, 1)   # 40x40 halo: no 2 stages
