"""Stride-2 forward convolutions on 8 or 16 input channels as compact phase-halo launches (cis_conv_s2_phase_plan, the host-side
rewrite cis_conv_igemm applies to such gather launches), on the CPU-built launch plans of the benchmarked step (256x448, batch 4) and of
the reference defaults (192x384, batch 16): which launches take it, the phase coordinates of their taps, the compact tap pairs and halo
planes (csrc/conv_igemm.cu: halo_step_off, thin_halo_load) and the K columns of the row pack every K=16 step reads, restated in numpy."""
import ctypes as C

import numpy as np
import pytest

from unsupervised_detection_b200 import _lib, engine
from unsupervised_detection_b200.step_graph import CISGraph


@pytest.fixture(scope='module', params=[(256, 448, 4), (192, 384, 16)], ids=['256x448x4', '192x384x16'])
def graph(request):
    H, W, B = request.param
    return CISGraph(H, W, B, device='cpu', global_batch=B)


def _plan(d):
    h, wk = _lib.CisConv(), (C.c_int16 * (2 * 49))()
    ok = _lib.load().cis_conv_s2_phase_plan(C.byref(d), C.byref(h), wk)
    return (h, list(wk)) if ok else None


def _channels(d):
    return sum(d.src[i].chunks for i in range(d.nsrc)) * 8


def _stride2_launches(g):
    """(gather descriptor, its ConvLayer) of every stride-2 forward launch of the plans."""
    layers = {}
    for plan in (g.fwd, g.bwd['G'], g.bwd['R']):
        for obj in plan.keep:
            if isinstance(obj, engine.ConvLayer) and obj.fwd_pack is not None:
                layers[obj.fwd_pack.w.data_ptr()] = obj
    for plan in (g.fwd, g.bwd['G'], g.bwd['R']):
        for fn, a, name, fl, lane in plan.ops:
            d = a[0]._obj if name == 'cis_conv_igemm' else None
            if d is not None and not d.halo and d.sh == 2:
                yield d, layers[d.wpack]


def _phase_of(h, t):
    return max(q for q in range(4) if h.ph_tap[q] <= t)


def _geometry(h):
    """(Wh, HP, plane bytes) of the compact halo of a launch."""
    wh, hh = 8 + h.ex, 16 * h.MT + h.ey
    return wh, wh * hh, (wh * hh * 16 + 127) // 128 * 128


def test_thin_stride2_launches_take_the_phase_halo(graph):
    """Only stride-2 launches on 8 or 16 channels are rewritten, into nph = 4 compact launches of the same taps, and only grids of at least
    296 16x8 tiles (the persistent kernel's); the recover 7x7 / 5x5 encoders and PWC-Net's first level are among them."""
    shapes = set()
    for d, layer in _stride2_launches(graph):
        ch, r = _channels(d), _plan(d)
        assert r is None or ch <= 16, (layer.name, ch)
        if r is None:
            continue
        h, _ = r
        assert h.N * -(-h.OW // 8) * -(-h.OH // (16 * h.MT)) * h.n_tiles >= 296
        assert h.halo == 1 and h.nph == 4 and h.thin == ch and h.sh == h.sw == 1 and h.dil == 1 and h.ntaps == d.ntaps
        assert (h.wpack, h.K_pad, h.BN, h.n_tiles, h.H, h.W, h.OH, h.OW) == (d.wpack, d.K_pad, d.BN, d.n_tiles, d.H, d.W, d.OH, d.OW)
        assert 1 <= h.MT <= 4 and h.MT * h.BN <= 128
        shapes.add((layer.k, ch))
    assert {(7, 8), (5, 16), (3, 8)} <= shapes, shapes


def _orig_taps(d, h):
    """Gather tap index of every tap of the phase launch, after checking that each tap (u, v) of the gather launch appears exactly once,
    in phase (u mod 2, v mod 2) at (u // 2 - hoy, v // 2 - hox), the phases one after the other."""
    where = {}
    for t in range(h.ntaps):
        where.setdefault((_phase_of(h, t), h.dh[t] + h.hoy, h.dw[t] + h.hox), []).append(t)
    orig = [None] * h.ntaps
    for t in range(d.ntaps):
        u, v = d.dh[t], d.dw[t]
        (i,) = where[((u % 2) * 2 + v % 2, u // 2, v // 2)]
        orig[i] = t
    assert h.ph_tap[0] == 0 and h.ph_tap[4] == h.ntaps and all(h.ph_tap[q] <= h.ph_tap[q + 1] for q in range(4))
    assert all(0 <= h.dh[t] <= h.ey and 0 <= h.dw[t] <= h.ex for t in range(h.ntaps))
    return orig


def test_phase_taps_restate_the_stride2_conv(graph):
    for d, layer in _stride2_launches(graph):
        r = _plan(d)
        if r is not None:
            assert sorted(_orig_taps(d, r[0])) == list(range(d.ntaps)), layer.name


def test_compact_phase_steps_stay_inside_the_planes(graph):
    """Every K=16 step's two core-matrix columns lie inside the 4 x thin/8 planes for all rows of every stacked tile; a tap pair (which
    may span two phases: the later phase's planes come later) has LBO > 0, only an odd last tap pairs with itself (LBO 0).  The halo
    stage, the pixel table and two weight stages fit the dynamic shared memory the launcher allows."""
    for d, layer in _stride2_launches(graph):
        r = _plan(d)
        if r is None:
            continue
        h, _ = r
        wh, hp, plane = _geometry(h)
        npl = h.thin // 8
        off = [_phase_of(h, t) * npl * plane + (h.dh[t] * wh + h.dw[t]) * 16 for t in range(h.ntaps)]
        if h.thin == 16:
            steps = [(o, plane) for o in off]
        else:
            steps = [(off[t], (off[t + 1] if t + 1 < h.ntaps else off[t]) - off[t]) for t in range(0, h.ntaps, 2)]
        footprint = (4 * npl - 1) * plane + hp * 16
        for s, (start, lbo) in enumerate(steps):
            pair = h.thin == 16 or 2 * s + 1 < h.ntaps
            assert (lbo > 0) if pair else (lbo == 0), (layer.name, s, lbo)
            assert lbo % 16 == 0 and start % 16 == 0 and lbo < (1 << 18) and start < (1 << 18)
            last_row = start + (16 * h.MT - 1) * wh * 16 + 7 * 16 + lbo
            assert last_row + 16 <= footprint, (layer.name, start, lbo, footprint)
        stage = -(-(4 * npl * plane) // 1024) * 1024
        assert stage + hp * 4 + 1024 + 2 * h.BN * 32 <= 226 * 1024, (layer.name, stage)


def test_row_pack_columns_of_every_step(graph):
    """kgroup j of K=16 step s reads the row-pack K columns of tap 2s + j (thin 8; past the last tap: column K_pad, outside the pack, which
    the TMA engine zero-fills) or channels 8j .. 8j + 7 of tap s (thin 16).  The dot product over those columns of the layer's row pack
    (K = tap * cin8 + channel, engine.ConvLayer.fwd_kmap) and the phase launch's taps equals the direct tap sum of its weights."""
    rng = np.random.default_rng(0)
    for d, layer in _stride2_launches(graph):
        r = _plan(d)
        if r is None:
            continue
        h, wk = r
        orig = _orig_taps(d, h)
        cin8, BN, nt = h.thin, h.BN, h.ntaps
        nst = (nt + 1) // 2 if cin8 == 8 else nt
        for s in range(nst):
            for j in range(2):
                t = 2 * s + j if cin8 == 8 else s
                want = (orig[t] * 8 if t < nt else d.K_pad) if cin8 == 8 else orig[t] * 16 + 8 * j
                assert wk[2 * s + j] == want, (layer.name, s, j)
        kmap = layer.fwd_kmap.numpy()
        w = rng.standard_normal(layer.k * layer.k * layer.cin * layer.cout).astype(np.float32)
        cols = min(BN, layer.cout)
        rows = np.zeros((d.K_pad, BN), np.float32)                  # the row pack of n-tile 0, transposed: [K][n]
        for k in range(d.K_pad):
            if kmap[k] >= 0:
                rows[k, :cols] = w[kmap[k] + np.arange(cols)]
        x = rng.standard_normal((d.ntaps, cin8)).astype(np.float32)   # the input a pixel sees through gather tap t
        got = np.zeros(BN)
        for s in range(nst):
            for j in range(2):
                t = 2 * s + j if cin8 == 8 else s
                a = x[orig[min(t, nt - 1)], slice(0, 8) if cin8 == 8 else slice(8 * j, 8 * j + 8)]
                k0 = wk[2 * s + j]
                b = rows[k0:k0 + 8] if k0 < d.K_pad else np.zeros((8, BN), np.float32)
                got += a @ b
        ref = np.zeros(BN)
        for t in range(d.ntaps):
            for c in range(cin8):
                ref += x[t, c] * rows[t * cin8 + c]
        np.testing.assert_allclose(got, ref, rtol=1e-4, atol=1e-4, err_msg=layer.name)
