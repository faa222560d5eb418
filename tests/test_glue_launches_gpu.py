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

The conv launches run unchecked here (tests/test_conv_launches_gpu.py checks them per launch).  One summary line per label (count, worst
bound ratio) is printed with pytest -s.  Measured worst ratios on an H100 80GB HBM3, over all graphs and direct calls: 0 for every
bit-exact kind; 0.996 for the bf16 resize-concat (x2, generic), its transposes (same, x2, generic), the nearest x2 transpose, the bf16
resize pair and the generator input; 0.994 cis_resize_f32_bwd_to_bf16_scaled; 0.993 cis_warp_costvol_bwd; 0.984 the direct
cis_warp_costvol_bwd_r at r = 1, 2, 3 (gate_one controls 4.5e4 - 1.0e5); 0.992 cis_warp_costvol; 0.154 cis_resize_bilinear_f32;
0.009 the dact_colsum partials; 0.001 cis_colsum; 0.0004 cis_flow_stats.  The bf16 kinds sit at the rounding term 2^-8 |ref|.  The whole
file runs in about 16 s."""
import pytest
import torch

import conv_launch_ref as R
import glue_launch_ref as G
from oracle import params as OP
from unsupervised_detection_b200 import _lib, engine as E
from unsupervised_detection_b200.models import functional as FN
from unsupervised_detection_b200.step_graph import CISGraph
from test_glue_launches_cpu import CONFIG2, PWC_BWD, FLOW_GIVEN

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]


def _report(key, glue):
    for lab, v in glue.summary().items():
        print('%-22s %-40s count %4d  worst bound ratio %.3g' % (key, lab, v['count'], v['worst']))
    if glue.controls is not None:
        print('%-22s negative controls (ratio > 1 = rejected): %s' % (key, glue.controls))


def _replay(plans, controls=False):
    glue = G.Glue(controls=controls)
    w = R.Walker(R.Recorder(), glue=glue)
    counts = {}
    for name, plan in plans:
        n = sum(glue.counts.values())
        before = dict(glue.counts)
        w.run(plan)
        counts[name] = {k: v - before.get(k, 0) for k, v in glue.counts.items() if v - before.get(k, 0)}
        assert sum(glue.counts.values()) - n == sum(counts[name].values())
    return glue, counts


def _config2_graph(masks=None):
    g = CISGraph(256, 448, 4, with_pwc=True, train=True, masks=masks)
    g.load_params(OP.make_params(seed=1, jitter=0.1))
    for pl in (g.pack_pwc, g.pack_gen, g.pack_rec):
        pl.run()
    gen = torch.Generator().manual_seed(7)
    img1 = R.smooth(4, 384, 640, 3, 0.25, gen).clamp(-0.5, 0.5)
    g.img1.copy_(img1)
    g.img2.copy_(torch.roll(img1, shifts=(2, 3), dims=(1, 2)) + 0.01 * torch.randn(4, 384, 640, 3, generator=gen))
    return g


@pytest.fixture(scope='module')
def config2():
    g = _config2_graph()
    glue, counts = _replay([('fwd', g.fwd), ('bwd_R', g.bwd['R']), ('bwd_G', g.bwd['G'])], controls=True)
    _report('config2_256x448_b4', glue)
    return dict(g=g, glue=glue, counts=counts)


def test_config2_every_glue_launch(config2):
    f = config2['glue'].failures
    assert not f, '\n'.join(f[:20])


def test_config2_launch_counts(config2):
    assert config2['counts'] == CONFIG2


def test_negative_controls_are_rejected(config2):
    c = config2['glue'].controls
    for kind in ('resize.row_off_by_one', 'rc_bwd.fold_dropped', 'rc_bwd.overwrite', 'dact.d_at_y', 'colsum.block_dropped',
                 'warp_costvol.fs_x1.25', 'tile.cis_warp_costvol', 'tile.cis_resize_concat_bf16.x2'):
        assert kind in c, (kind, c)
        assert c[kind] > 1.0, (kind, c)


def test_pwc_runner_every_glue_launch():
    B, H, W = 2, 384, 640
    r = FN._PWCRunner(B, H, W, 'cuda', 'pwcnet', trainable=True)
    r.ensure_backward()
    r.reload(OP.make_params(seed=1, jitter=0.1))
    gen = torch.Generator().manual_seed(13)
    img1 = R.smooth(B, H, W, 3, 0.25, gen).clamp(-0.5, 0.5)
    r.img1.copy_(img1)
    r.img2.copy_(torch.roll(img1, shifts=(2, 3), dims=(1, 2)) + 0.01 * torch.randn(B, H, W, 3, generator=gen))
    r.dflow_out.copy_(R.smooth(B, H, W, 2, 1.0, gen))
    glue, counts = _replay([('fwd', r.bld.fwd), ('bwd', r.bwd)], controls=True)
    _report('pwc_runner_384x640_b2', glue)
    assert counts['bwd'] == PWC_BWD
    assert not glue.failures, '\n'.join(glue.failures[:20])


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
    glue = _direct([('cis_warp_costvol_bwd', (c1.data_ptr(), C, 0, c2.data_ptr(), C, 0, flow.data_ptr(), 2.5, B, h, w, C, dcorr.data_ptr(),
                                              88, 0, dc1.data_ptr(), C, 0, dc2.data_ptr(), C, 0, dfl.data_ptr(), 8, 0, 0, gs.data_ptr(),
                                              ws.data_ptr(), ds.data_ptr()))])
    _report('direct_costvol_bwd', glue)
    assert not glue.failures, '\n'.join(glue.failures[:20])
    assert glue.controls['costvol_bwd.gate_one'] > 1.0, glue.controls


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
    glue = _direct([('cis_warp_costvol_bwd_r', args)])
    _report('direct_costvol_bwd_r%d' % r, glue)
    assert glue.counts['cis_warp_costvol_bwd_r'] == 1
    assert not glue.failures, '\n'.join(glue.failures[:20])
    assert glue.controls['costvol_bwd.gate_one'] > 1.0, glue.controls


def _flow_given(H, W, B, seed):
    g = CISGraph(H, W, B, with_pwc=False, train=True)
    g.load_params(OP.make_params(seed=4, jitter=0.1, nets=('MaskNet', 'FlownetS')))
    for pl in (g.pack_gen, g.pack_rec):
        pl.run()
    gen = torch.Generator().manual_seed(seed)
    g.image.copy_(torch.rand(B, H, W, 3, generator=gen) - 0.5)
    g.flow.copy_(R.smooth(B, H, W, 2, 0.3, gen))
    return g


def test_defaults_192x384_batch16_every_glue_launch():
    g = _flow_given(192, 384, 16, 3)
    glue, counts = _replay([('fwd', g.fwd), ('bwd_R', g.bwd['R']), ('bwd_G', g.bwd['G'])])
    _report('defaults_192x384_b16', glue)
    assert counts == FLOW_GIVEN
    assert not glue.failures, '\n'.join(glue.failures[:20])


def test_odd_100x172_batch3_generic_resize():
    g = _flow_given(100, 172, 3, 5)
    glue, counts = _replay([('fwd', g.fwd), ('bwd_R', g.bwd['R']), ('bwd_G', g.bwd['G'])])
    _report('odd_100x172_b3', glue)
    assert counts == FLOW_GIVEN
    assert not glue.failures, '\n'.join(glue.failures[:20])
    s = glue.summary()
    assert s['cis_resize_concat_bf16.generic']['count'] >= 6
    assert s['cis_resize_concat_bf16_bwd.generic']['count'] >= 12


# ------------------------------------------------------------------------------------------------------------ direct calls
def _bf(gen, *shape):
    return torch.randn(*shape, generator=gen).to(torch.bfloat16).cuda()


def _direct(ops):
    plan = E.Plan('direct')
    for name, args in ops:
        plan.add(name, *args)
    glue, _ = _replay([('direct', plan)], controls=True)
    return glue


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
    glue = _direct([('cis_resize_concat_bf16', (srcs, 2, N, H, W, dst.data_ptr(), 48, 8, OH, OW)),
                    ('cis_resize_concat_bf16_bwd', (dd.data_ptr(), 40, 16, N, OH, OW, grads, want, acc, 2, H, W))])
    _report('direct_rc_%dx%d_%dx%d' % (H, W, OH, OW), glue)
    assert not glue.failures, '\n'.join(glue.failures[:20])
    assert glue.counts['cis_resize_concat_bf16_bwd'] == 1
    assert glue.controls['rc_bwd.fold_dropped'] > 1.0 and glue.controls['rc_bwd.overwrite'] > 1.0, glue.controls


def test_direct_add_slice_forms():
    """The three forms of cis_add_slice: residual gradient with and without accumulate (reps = 1), the zeroing of a parity no tap reaches
    (reps = 0, source = destination), and the 3-call fold of shared features (reps = 3) accumulating.  The step itself only copies."""
    gen = torch.Generator().manual_seed(17)
    n = 4 * 9 * 13
    dst = [_bf(gen, n, 24) for _ in range(4)]
    src = _bf(gen, 3 * n, 16)
    glue = _direct([('cis_add_slice', (dst[0].data_ptr(), 24, 8, src.data_ptr(), 16, 0, n, 2, 1, 1)),
                    ('cis_add_slice', (dst[1].data_ptr(), 24, 0, src.data_ptr(), 16, 8, n, 1, 1, 0)),
                    ('cis_add_slice', (dst[2].data_ptr(), 24, 16, dst[2].data_ptr(), 24, 16, n, 1, 0, 0)),
                    ('cis_add_slice', (dst[3].data_ptr(), 24, 8, src.data_ptr(), 16, 0, n, 2, 3, 1))])
    _report('direct_add_slice', glue)
    assert not glue.failures, '\n'.join(glue.failures[:20])
    assert {k: v['count'] for k, v in glue.summary().items()} == {'cis_add_slice.accumulate': 2, 'cis_add_slice.copy': 1,
                                                                 'cis_add_slice.zero': 1}
    assert glue.controls['add_slice.acc_dropped'] > 1.0


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
    glue = _direct(ops)
    _report('direct_bf16_resize', glue)
    assert not glue.failures, '\n'.join(glue.failures[:20])
    assert glue.counts['cis_resize_bilinear_bf16'] == 2 and glue.counts['cis_resize_bilinear_bf16_bwd'] == 2
    assert glue.controls['tile.cis_resize_bilinear_bf16'] > 1.0


# ------------------------------------------------------------------------------------------------------------ poisoned replay
def _targets(g, plans):
    """(Acts, fp32 / fp64 scratch tensors, bf16 scratch tensors) the plans of g write: see _poison."""
    acts, f32, b16, seen = [], [], [], set()

    def walk(o):
        if o is None or id(o) in seen:
            return
        seen.add(id(o))
        if isinstance(o, E.Act):
            acts.append(o)
            walk(o.grad)
        elif isinstance(o, torch.Tensor):
            if o.dtype in (torch.float32, torch.float64) and o.is_cuda:
                f32.append(o)
        elif isinstance(o, (list, tuple)):
            for x in o:
                walk(x)
        elif isinstance(o, dict):
            for x in o.values():
                walk(x)
        elif isinstance(o, E.ConvLayer):
            walk(o.dcat)
            walk(o.dwp)
            walk(o.colpart)
            walk(o.dwp_hi)
            for pk in o.tr_packs or ():
                walk(pk.dwp)
            if o.tr_planes is not None:
                b16.append(o.tr_planes)
    walk(g.bld.keep)
    for p in plans:
        walk(p.keep)
    for L in list(g.gen.all_layers()) + list(g.rec.all_layers()) + (list(g.pwc.all_layers()) if g.with_pwc else []):
        walk(L)
    # scalars[5:8] are slots no kernel writes (cis_cis_loss_reduce defines [0, 5))
    named = [g.image, g.flow, g.mask, g.flow1, g.pred, g.dmask, g.sums, g.scalars[:5], g.coef]
    named += [t for t in (getattr(g, 'dpred', None), getattr(g, 'stats', None), getattr(g, 'image_st', None), getattr(g, 'flow_st', None))
              if t is not None]
    if g.with_pwc:
        named.append(g.flow_full)
    # what a batch upload writes (the two buffers of a staged graph, image and flow otherwise) is input, not poisoned
    inputs = {t.data_ptr() for t in (g.inputs if g.staged else (g.image, g.flow))}
    named = [t for t in named if t.data_ptr() not in inputs]
    full = {t.data_ptr() for t in named}
    f32 = named + [t for t in f32 if t.data_ptr() not in inputs and t.data_ptr() not in full]
    return acts, f32, b16


def _poison(g, modes, sentinel):
    acts, f32, b16 = _targets(g, [g.fwd] + [g.bwd[m] for m in modes])
    for a in acts:
        idx = [a.c_off + p for p, m in enumerate(a.chanmap) if m >= 0]
        if not idx:
            continue
        v = torch.full((a.N, a.H, a.W, len(idx)), sentinel, dtype=torch.bfloat16, device='cuda')
        if sentinel == sentinel:
            v[..., 1::2] = -sentinel
        a.buf[:a.N].index_copy_(3, torch.tensor(idx, device='cuda'), v)
    for t in f32 + b16:
        t.fill_(sentinel)
        if sentinel == sentinel:
            t.view(-1)[1::2] = -sentinel
    for m in modes:
        st = g.store(m)
        for name, _, n, off, _ in st.entries:
            st.grad[off:off + n].fill_(sentinel)


def _outputs(g, modes):
    out = {k: getattr(g, k).clone() for k in ('mask', 'flow1', 'pred', 'sums')}
    out['scalars'] = g.scalars[:5].clone()
    for m in modes:
        out['grad_' + m] = g.store(m).grad.clone()
    return out


def _bits(t):
    return t.view(torch.int32 if t.element_size() == 4 else torch.int64)


@pytest.mark.parametrize('which', ['config2', 'boxes'])
def test_poisoned_replay_reads_only_what_it_wrote(which):
    """Clean run from the fresh graph, then every intermediate buffer (Act real channels, dcat, parity planes, weight-gradient slices,
    partial sums, fp32 scratch, the real entries of the flat gradients) filled with NaN, then with +-2^100, and the same plans rerun on
    the same inputs and parameters: every output and gradient must be bit-identical to the clean run."""
    g = _config2_graph(masks='boxes' if which == 'boxes' else None)
    modes = ['R'] if which == 'boxes' else ['R', 'G']
    plans = [g.fwd] + [g.bwd[m] for m in modes]
    for p in plans:
        p.run()
    torch.cuda.synchronize()
    clean = _outputs(g, modes)
    for sentinel in (float('nan'), 2.0 ** 100):
        _poison(g, modes, sentinel)
        torch.cuda.synchronize()
        for p in plans:
            p.run()
        torch.cuda.synchronize()
        now = _outputs(g, modes)
        bad = [k for k in clean if not torch.equal(_bits(now[k]), _bits(clean[k]))]
        if bad:
            # name the first launch that read a non-finite operand
            _poison(g, modes, float('nan'))
            glue = G.Glue()
            w = R.Walker(R.Recorder(), glue=glue)
            for p in plans:
                w.run(p)
            pytest.fail('sentinel %r: %s differ from the clean run; first glue launch reading a non-finite operand: %s'
                        % (sentinel, bad, glue.first_nonfinite))
