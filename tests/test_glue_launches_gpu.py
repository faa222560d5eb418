"""Every non-convolution launch of the benchmarked train step and of PWC-Net's backward, at its benchmarked shape and launch plan, against a
float64 reference of the same launch (tests/glue_launch_ref.py: argument decoding, references, bounds and their derivation), and a
poisoned-buffer replay showing that each plan reads only what it wrote.

  config 2     the train graph at 256x448, batch 4, PWC-Net at 384x640: fwd, bwd['R'], bwd['G'], with the negative controls
  PWC-Net      _PWCRunner(2, 384, 640, trainable=True) fwd and bwd: the five warp + cost-volume transposes, 91 dact_colsum, 8 parity splits
  defaults     192x384, batch 16, flow given directly
  odd          100x172, batch 3, flow given: the generic (non-x2) resize-concat and its transpose
  direct       the branches no graph reaches: the nx > 8 fallback of the resize-concat transpose, 1-pixel sources, 3 replicas with
               accumulate, the bf16 resize pair at a non-binary ratio; the warp + cost-volume transpose on independent random features
               (about half the correlations negative, so the leaky gate shows) at R = 4 and, through cis_warp_costvol_bwd_r, at r = 1, 2, 3

Each graph is replayed once, with its conv launches checked in the same replay (launch_suites.walk_graph, shared with
tests/test_conv_launches_gpu.py).  One summary line per label (count, worst bound ratio) is printed with pytest -s.  Measured worst ratios
on an H100 80GB HBM3, over all graphs and direct calls: 0 for every bit-exact kind; 0.996 for the bf16 resize-concat (x2, generic), its
transposes (same, x2, generic), the nearest x2 transpose, the bf16 resize pair and the generator input; 0.994
cis_resize_f32_bwd_to_bf16_scaled; 0.993 cis_warp_costvol_bwd; 0.984 the direct cis_warp_costvol_bwd_r at r = 1, 2, 3 (gate_one controls
4.5e4 - 1.0e5); 0.992 cis_warp_costvol; 0.154 cis_resize_bilinear_f32; 0.009 the dact_colsum partials; 0.001 cis_colsum; 0.0004
cis_flow_stats.  The bf16 kinds sit at the rounding term 2^-8 |ref|."""
import pytest
import torch

import conv_launch_ref as R
from launch_suites import CONFIG2, FLOW_GIVEN, PWC_BWD, assert_within_bounds, bits, build, load_inputs, poison_cis, report, walk_graph, \
    walk_plans
from unsupervised_detection_b200 import _lib, engine as E

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]


def test_config2_every_glue_launch():
    assert_within_bounds(walk_graph('config2'))


def test_config2_launch_counts():
    assert walk_graph('config2')['counts'] == CONFIG2


def test_negative_controls_are_rejected():
    c = walk_graph('config2')['controls']
    for kind in ('resize.row_off_by_one', 'rc_bwd.fold_dropped', 'rc_bwd.overwrite', 'dact.d_at_y', 'colsum.block_dropped',
                 'warp_costvol.fs_x1.25', 'tile.cis_warp_costvol', 'tile.cis_resize_concat_bf16.x2'):
        assert kind in c, (kind, c)
        assert c[kind] > 1.0, (kind, c)


def test_pwc_runner_every_glue_launch():
    r = walk_graph('pwc_runner')
    assert r['counts']['bwd'] == PWC_BWD
    assert_within_bounds(r)


def test_direct_warp_costvol_bwd_gate():
    """Independent random features, so that about half the correlations are negative: the transpose with a flow, and the control that
    takes the leaky gate as 1 everywhere (the pyramid's correlations are almost all positive, where the gate hardly shows)."""
    gen = torch.Generator().manual_seed(23)
    B, h, w, C = 1, 12, 20, 16
    c1, c2 = _bf(gen, B, h, w, C), _bf(gen, B, h, w, C)
    flow = R.smooth(B, h, w, 2, 1.5, gen, div=4).cuda()
    dcorr = _bf(gen, B, h, w, 88)
    dc1, dc2, dfl = (torch.zeros(B, h, w, n, dtype=torch.bfloat16, device='cuda') for n in (C, C, 8))
    npix = B * h * w
    gs, ws = torch.zeros(npix * 81, device='cuda'), torch.zeros(npix * C, device='cuda')
    ds = torch.zeros(npix * C, dtype=torch.float64, device='cuda')
    args = (c1.data_ptr(), C, 0, c2.data_ptr(), C, 0, flow.data_ptr(), 2.5, B, h, w, C, dcorr.data_ptr(), 88, 0, dc1.data_ptr(), C, 0,
            dc2.data_ptr(), C, 0, dfl.data_ptr(), 8, 0, 0, gs.data_ptr(), ws.data_ptr(), ds.data_ptr())
    out = _direct('direct_costvol_bwd', [('cis_warp_costvol_bwd', args)])
    assert out['controls']['costvol_bwd.gate_one'] > 1.0, out['controls']


@pytest.mark.parametrize('r', [1, 2, 3])
def test_direct_warp_costvol_bwd_r_gate(r):
    """The same for the search-range entry point cis_warp_costvol_bwd_r: the PWC-Net graphs at ranges 1-3 hardly show the gate, so here
    the gate_one control shows that the bound rejects a wrong transpose at each range."""
    gen = torch.Generator().manual_seed(23 + r)
    B, h, w, C = 1, 12, 20, 16
    nd = (2 * r + 1) ** 2
    pad = 8 * (-(-nd // 8))
    c1, c2 = _bf(gen, B, h, w, C), _bf(gen, B, h, w, C)
    flow = R.smooth(B, h, w, 2, 1.5, gen, div=4).cuda()
    dcorr = _bf(gen, B, h, w, pad)
    dc1, dc2, dfl = (torch.zeros(B, h, w, n, dtype=torch.bfloat16, device='cuda') for n in (C, C, 8))
    npix = B * h * w
    gs, ws = torch.zeros(npix * nd, device='cuda'), torch.zeros(npix * C, device='cuda')
    ds = torch.zeros(npix * C, dtype=torch.float64, device='cuda')
    args = (c1.data_ptr(), C, 0, c2.data_ptr(), C, 0, flow.data_ptr(), 2.5, B, h, w, C, dcorr.data_ptr(), pad, 0, dc1.data_ptr(), C, 0,
            dc2.data_ptr(), C, 0, dfl.data_ptr(), 8, 0, 0, gs.data_ptr(), ws.data_ptr(), ds.data_ptr(), r)
    out = _direct('direct_costvol_bwd_r%d' % r, [('cis_warp_costvol_bwd_r', args)])
    assert out['counts']['direct']['cis_warp_costvol_bwd_r'] == 1
    assert out['controls']['costvol_bwd.gate_one'] > 1.0, out['controls']


def test_defaults_192x384_batch16_every_glue_launch():
    r = walk_graph('defaults')
    assert r['counts'] == FLOW_GIVEN
    assert_within_bounds(r)


def test_odd_100x172_batch3_generic_resize():
    r = walk_graph('odd')
    assert r['counts'] == FLOW_GIVEN
    assert_within_bounds(r)
    s = r['summary']
    assert s['cis_resize_concat_bf16.generic']['count'] >= 6
    assert s['cis_resize_concat_bf16_bwd.generic']['count'] >= 12


# ------------------------------------------------------------------------------------------------------------ direct calls
def _bf(gen, *shape):
    return torch.randn(*shape, generator=gen).to(torch.bfloat16).cuda()


def _direct(key, ops):
    """The ops as one plan, every launch checked with the negative controls -> walk_plans' result, reported under `key`."""
    plan = E.Plan('direct')
    for name, args in ops:
        plan.add(name, *args)
    r = walk_plans(R.Recorder(), [('direct', plan)], glue_controls=True)
    report(key, r['summary'], r['controls'])
    assert_within_bounds(r)
    return r


@pytest.mark.parametrize('H,W,OH,OW', [(3, 4, 14, 17), (1, 5, 3, 9), (6, 1, 11, 2), (5, 7, 9, 13)])
def test_direct_resize_concat_pair(H, W, OH, OW):
    """Two sources, one batch-broadcast with 3 replicas; the transpose accumulates into both.  3x4 -> 14x17 takes the nx > 8 fallback of
    the transpose; 1-pixel sources clamp `hi`."""
    gen = torch.Generator().manual_seed(H * 100 + W)
    N, nm = 6, 2
    s0, s1 = _bf(gen, N, H, W, 16), _bf(gen, nm, H, W, 24)
    dst = torch.zeros(N, OH, OW, 48, dtype=torch.bfloat16, device='cuda')
    srcs = (_lib.CisSrc * 2)(_lib.CisSrc(s0.data_ptr(), 16, 8, 1, 0), _lib.CisSrc(s1.data_ptr(), 24, 0, 2, nm))
    dd = _bf(gen, N, OH, OW, 40)
    g0, g1 = _bf(gen, N, H, W, 16), _bf(gen, nm, H, W, 24)
    grads = (_lib.CisSrc * 2)(_lib.CisSrc(g0.data_ptr(), 16, 8, 1, 0), _lib.CisSrc(g1.data_ptr(), 24, 0, 2, nm))
    want, acc = (_lib.C.c_int32 * 2)(1, 1), (_lib.C.c_int32 * 2)(1, 1)
    out = _direct('direct_rc_%dx%d_%dx%d' % (H, W, OH, OW),
                  [('cis_resize_concat_bf16', (srcs, 2, N, H, W, dst.data_ptr(), 48, 8, OH, OW)),
                   ('cis_resize_concat_bf16_bwd', (dd.data_ptr(), 40, 16, N, OH, OW, grads, want, acc, 2, H, W))])
    assert out['counts']['direct']['cis_resize_concat_bf16_bwd'] == 1
    assert out['controls']['rc_bwd.fold_dropped'] > 1.0 and out['controls']['rc_bwd.overwrite'] > 1.0, out['controls']


def test_direct_add_slice_forms():
    """The three forms of cis_add_slice: residual gradient with and without accumulate (reps = 1), the zeroing of a parity no tap reaches
    (reps = 0, source = destination), and the 3-call fold of shared features (reps = 3) accumulating.  The step itself only copies."""
    gen = torch.Generator().manual_seed(17)
    n = 4 * 9 * 13
    dst = [_bf(gen, n, 24) for _ in range(4)]
    src = _bf(gen, 3 * n, 16)
    out = _direct('direct_add_slice', [('cis_add_slice', (dst[0].data_ptr(), 24, 8, src.data_ptr(), 16, 0, n, 2, 1, 1)),
                                       ('cis_add_slice', (dst[1].data_ptr(), 24, 0, src.data_ptr(), 16, 8, n, 1, 1, 0)),
                                       ('cis_add_slice', (dst[2].data_ptr(), 24, 16, dst[2].data_ptr(), 24, 16, n, 1, 0, 0)),
                                       ('cis_add_slice', (dst[3].data_ptr(), 24, 8, src.data_ptr(), 16, 0, n, 2, 3, 1))])
    assert {k: v['count'] for k, v in out['summary'].items()} == {'cis_add_slice.accumulate': 2, 'cis_add_slice.copy': 1,
                                                                 'cis_add_slice.zero': 1}
    assert out['controls']['add_slice.acc_dropped'] > 1.0


def test_direct_bf16_resize_pair():
    """cis_resize_bilinear_bf16 / _bwd (accumulating) at non-binary ratios, up and down."""
    gen = torch.Generator().manual_seed(11)
    ops = []
    keep = []
    for (H, W, OH, OW) in ((5, 7, 9, 13), (13, 22, 7, 11)):
        src = _bf(gen, 3, H, W, 24)
        dst = torch.zeros(3, OH, OW, 16, dtype=torch.bfloat16, device='cuda')
        dd = _bf(gen, 3, OH, OW, 16)
        ds = _bf(gen, 3, H, W, 24)
        keep += [src, dst, dd, ds]
        ops += [('cis_resize_bilinear_bf16', (src.data_ptr(), 24, 8, 3, H, W, dst.data_ptr(), 16, 0, OH, OW, 2)),
                ('cis_resize_bilinear_bf16_bwd', (dd.data_ptr(), 16, 0, 3, OH, OW, ds.data_ptr(), 24, 8, H, W, 2, 1))]
    out = _direct('direct_bf16_resize', ops)
    assert out['counts']['direct']['cis_resize_bilinear_bf16'] == 2 and out['counts']['direct']['cis_resize_bilinear_bf16_bwd'] == 2
    assert out['controls']['tile.cis_resize_bilinear_bf16'] > 1.0


# ------------------------------------------------------------------------------------------------------------ poisoned replay
def _outputs(g, modes):
    out = {k: getattr(g, k).clone() for k in ('mask', 'flow1', 'pred', 'sums')}
    out['scalars'] = g.scalars[:5].clone()
    for m in modes:
        out['grad_' + m] = g.store(m).grad.clone()
    return out


@pytest.mark.parametrize('which', ['config2', 'boxes'])
def test_poisoned_replay_reads_only_what_it_wrote(which):
    """Clean run from the fresh graph, then every intermediate buffer (Act real channels, dcat, parity planes, weight-gradient slices,
    partial sums, fp32 scratch, the real entries of the flat gradients) filled with NaN, then with +-2^100, and the same plans rerun on
    the same inputs and parameters: every output and gradient must be bit-identical to the clean run."""
    g, _, _ = build(which, 'cuda')
    load_inputs(which, g)
    modes = list(g.bwd)
    plans = [g.fwd] + [g.bwd[m] for m in modes]
    for p in plans:
        p.run()
    torch.cuda.synchronize()
    clean = _outputs(g, modes)
    for sentinel in (float('nan'), 2.0 ** 100):
        poison_cis(g, modes, sentinel)
        torch.cuda.synchronize()
        for p in plans:
            p.run()
        torch.cuda.synchronize()
        now = _outputs(g, modes)
        bad = [k for k in clean if not torch.equal(bits(now[k]), bits(clean[k]))]
        if bad:
            # name the first launch that read a non-finite operand
            poison_cis(g, modes, float('nan'))
            first = walk_plans(R.Recorder(), [(p.name, p) for p in plans])['first_nonfinite']
            pytest.fail('sentinel %r: %s differ from the clean run; first glue launch reading a non-finite operand: %s'
                        % (sentinel, bad, first))
