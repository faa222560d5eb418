"""The compact thin-input halo format (CisConv.thin) on the CPU-built launch plan of the benchmarked step (256x448, batch 4): which
launches take it, the tap order its K=16 tap pairs need, the descriptor fields the kernel derives from it (csrc/conv_igemm.cu:
halo_step_off) and the K order of the pre-tiled weights (csrc/misc_kernels.cu: pack_weights_thin_body), restated in numpy."""
import numpy as np
import pytest

from unsupervised_detection_b200 import engine
from unsupervised_detection_b200.step_graph import CISGraph


@pytest.fixture(scope='module')
def graph():
    return CISGraph(256, 448, 4, device='cpu', global_batch=4)


def _halo_convs(g):
    for plan in (g.fwd, g.bwd['G'], g.bwd['R']):
        for fn, a, name, fl, lane in plan.ops:
            if name == 'cis_conv_igemm' and a[0]._obj.halo:
                yield a[0]._obj


def _subs(d):
    """(first tap, tap count) of every sub-problem of a launch."""
    return [(d.sub[i].tap0, d.sub[i].ntaps) for i in range(d.nsub)] if d.nsub > 1 else [(0, d.ntaps)]


def _steps(d, t0, nt):
    """halo_step_off: per K=16 step, (A start, LBO) in bytes."""
    wh, hp = 8 + d.ex, (8 + d.ex) * (16 * d.MT * max(d.nwg, 1) + d.ey)
    off = [(d.dh[t] * wh + d.dw[t]) * 16 for t in range(t0, t0 + nt)]
    if d.thin == 16:
        return [(o, (hp * 16 + 127) // 128 * 128) for o in off]
    return [(off[t], (off[t + 1] if t + 1 < nt else off[t]) - off[t]) for t in range(0, nt, 2)]


def test_compact_format_exactly_for_thin_undilated_halo_launches(graph):
    n = 0
    for d in _halo_convs(graph):
        ch = sum(d.src[i].chunks for i in range(d.nsrc)) * 8
        want = ch if ch <= 16 and d.dil == 1 and d.nph <= 1 else 0
        assert d.thin == want, (ch, d.dil, d.nph, d.thin)
        n += bool(d.thin)
    assert n >= 30            # the generator, recover and PWC-Net thin layers, forward and data gradient


def test_compact_descriptors_stay_inside_the_halo(graph):
    """Every K=16 step's two core-matrix columns (start, start + LBO) lie inside the staged planes for all 128 rows of every stacked tile;
    LBO and SBO are 16-byte multiples and LBO >= 0 (the taps of a pair are listed in increasing halo offset)."""
    for d in (d for d in _halo_convs(graph) if d.thin):
        wh, hh = 8 + d.ex, 16 * d.MT * max(d.nwg, 1) + d.ey
        planes = d.thin // 8
        plane = (wh * hh * 16 + 127) // 128 * 128
        footprint = (planes - 1) * plane + wh * hh * 16
        sbo = wh * 16
        for t0, nt in _subs(d):
            for start, lbo in _steps(d, t0, nt):
                assert lbo >= 0 and lbo % 16 == 0 and sbo % 16 == 0 and start % 16 == 0
                assert lbo < (1 << 18)                                   # the 14-bit LBO field, in 16-byte units
                last_row = start + (16 * d.MT * max(d.nwg, 1) - 1) * sbo + 7 * 16 + lbo    # 8 GEMM rows = 8 pixels of one halo row
                assert last_row + 16 <= footprint, (start, lbo, footprint)


def _thin_tiles(w_kt, thin, BN):
    """numpy restatement of pack_weights_thin_body for one n-tile: w_kt[tap][c][n] -> [step][BN * 16] bf16-element tiles."""
    nt, cin8, _ = w_kt.shape
    nst = (nt + 1) // 2 if thin == 8 else nt
    out = np.zeros((nst, BN * 16), np.float32)
    for s in range(nst):
        for n in range(BN):
            for j in range(2):
                for e in range(8):
                    t, c = (2 * s + j, e) if thin == 8 else (s, 8 * j + e)
                    if t < nt and c < cin8:
                        out[s, ((n // 8) * 2 + j) * 64 + (n % 8) * 8 + e] = w_kt[t, c, n]
    return out


@pytest.mark.parametrize('k,thin', [(3, 8), (5, 8), (7, 16), (3, 16), (2, 8)])
def test_tap_pair_k_order(k, thin):
    """The K order a K=16 step multiplies: A column kgroup j of step s is tap 2s + j channels 0-7 (thin 8) or tap s channels 8j .. 8j + 7
    (thin 16), in the tap order the planner lists (2 x 2 = the taps of one output parity of a stride-2 data gradient, listed there in
    decreasing offset).  The dot product over the packed tiles and the sorted taps equals the direct tap sum."""
    rng = np.random.default_rng(k * 100 + thin)
    taps = [(r, c) for r in range(k) for c in range(k)]
    if k == 2:
        taps = taps[::-1]
    cin8, BN = thin, 16
    w = rng.standard_normal((len(taps), cin8, BN)).astype(np.float32)
    x = rng.standard_normal((len(taps), cin8)).astype(np.float32)   # the input a pixel sees through each tap
    order = engine.thin_tap_order(thin, taps)
    offs = [taps[i][0] * 16 + taps[i][1] for i in order]
    assert offs == sorted(offs) or thin == 16
    tiles = _thin_tiles(w[order], thin, BN)
    xs = x[order]
    got = np.zeros(BN)
    for s in range(tiles.shape[0]):
        for j in range(2):
            t, cs = (2 * s + j, slice(0, 8)) if thin == 8 else (s, slice(8 * j, 8 * j + 8))
            a = xs[t, cs] if t < len(taps) else xs[t - 1, cs]       # an odd last step reads its own tap again against zero weights
            for n in range(BN):
                b = tiles[s, ((n // 8) * 2 + j) * 64 + (n % 8) * 8:((n // 8) * 2 + j) * 64 + (n % 8) * 8 + 8]
                got[n] += float(np.dot(a, b))
    ref = np.einsum('tc,tcn->n', x, w)
    np.testing.assert_allclose(got, ref, rtol=1e-5, atol=1e-5)
