"""Every launch of the PWC-Net training step (FlowTrainGraph), at train_flow.py's and tools/time_flow_train.py's shapes, checked on its
own against an fp64 reference: the conv launches by tests/conv_launch_ref.py, the others by tests/glue_launch_ref.py (the seven entry
points of the step -- multi-scale loss and its backward, the unsupervised loss and its backward, the augmentation's parameter draws and
per-pixel pass, TF-Adam with L2 -- and the glue the step shares with the inference graphs).  The graphs (tests/test_flow_train_launches_cpu.py
pins their launch census):

  default   FlowTrainGraph(192, 384, 16, in_hw=(384, 640)): frames resized on the device, loss targets at s0 = 0.5, s1 = 0.6
  unsup     the same with loss='unsupervised': network batch 32, the four packs into the halves of the image Acts
  timed     FlowTrainGraph(384, 640, 8): the timed step
  shard     FlowTrainGraph(192, 384, 4, global_batch=16, in_hw=(384, 640), loss='robust', options={'use_dense_cx': False}, augment=True,
            sample_offset=8): robust rho, the "sm" network, the augmentation, rank 2 of 4

Parameters are pwc_options_ref.make_params with a 0.1 jitter; frames are textured (smooth plus per-pixel noise), the ground truth a
smooth flow of several pixels at 384x640.  Two full steps (aug, fwd, bwd, adam, pack) are walked, each with a fresh Walker and
Glue(controls=True).  Step 2 checks the re-pack after Adam (the conv references read the updated fp32 master in both the forward and
the data-gradient orientation), Adam at t = 2 with non-zero m and v, and a redrawn augmentation.

After step 1's bwd walk the fwd_bwd CUDA graph of train_step(use_graph=True) is captured, every buffer the plans write (not the inputs,
parameters, m, v, step or lr) is filled with NaN, then with +-2^100, and the graph is replayed on the same state: the flat gradient and
the loss sums must be bit-identical to the walked step's.  Also: epe() at `default` against fp64 (the cis_crop_resize_flow_f32 resize of
the prediction to 384x640 with vectors scaled by (2, 5/3), and the cis_masked_epe sums), and cis_abs_sum against an fp64 sum.

One summary line per graph and label and the controls are printed with pytest -s.  Controls: every control made must be rejected
(ratio > 1) except costvol_bwd.gate_one (tests/test_graph_variants_launches_gpu.py says why).

At `unsup` the untrained network's two directions disagree almost everywhere, so its mask keeps only a few hundred of the 2.36 M pixels
per step.  test_unsup_loss_launches_on_partly_consistent_flows therefore also runs the two unsupervised launches on flows built to be
partly consistent, where the census, coef and gather references meet tens of thousands of visible pixels.

Measured with pytest -m gpu tests/test_flow_train_launches_gpu.py -s on an H100 80GB HBM3 (700 W power limit), the printed values:
every launch of both steps of the four graphs within its bound, no bug found.  Worst ratios over the graphs and steps:
cis_flow_multiscale_loss 0.0189, cis_flow_multiscale_loss_bwd 0.995 (the bf16 rounding term), cis_adam_l2 0.985 (timed, step 2),
cis_flow_aug_params 0 (every column the fp32 rounding of the fp64 draw), cis_flow_augment 0.152, cis_unsup_flow_loss 0.291 and
cis_unsup_flow_loss_bwd 0.325 (unsup; 0.272 and 0.690 on the partly consistent flows); epe() 1.54e-4; conv launches 0.99.  Masks:
at unsup 243 and 266 visible pixels (steps 1, 2), 0 differing from fp64, 0 within the occlusion test's epsilon; on the partly consistent
flows 61 876 visible of 294 912, 6 within epsilon, 0 differing.  Controls: ms_loss.axes_swapped 1.6e4 - 7.1e4, ms_loss.level_scale
3.0e5 - 4.0e5, ms_loss_bwd.weights_reversed 1.6e4, tile.cis_flow_multiscale_loss_bwd 8.6 - 9.0, unsup.mask_ones 3.3e35 (a direction whose
mask is empty: its photometric sum and bound are 0, so the FLOOR of 2^-100 divides the sum of psi, ~2.6e5) and 5.6e30 on the partly
consistent flows (coef at a masked pixel over the FLOOR), unsup_bwd.smooth_dropped 4.9e5 and 7.7e5, pack.unswapped 1.3e30,
aug_params.step_frozen inf (the accepted attempts differ), augment.flow_unmapped 1.8e5, adam.decay_everywhere 1.0e8 - 1.2e18,
adam.t_off_by_one 5.6e3.  Both poisoned replays bit-identical at every graph.  The file ran in 35 s: the four walks 7 - 10 s each."""
import time

import pytest
import torch

import conv_launch_ref as R
import glue_launch_ref as G
import pwc_options_ref as REF
from unsupervised_detection_b200 import _lib, engine as E
from test_flow_train_launches_cpu import CONV, GLUE, GRAPHS, KEYS, PLANS, build

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

UNREJECTED = {'costvol_bwd.gate_one'}


def _inputs(g, seed):
    """Textured frames in [-0.5, 0.5] (tests/test_unsup_flow_gpu.py's construction) and a smooth ground truth of several pixels, at the
    upload size."""
    gen = torch.Generator().manual_seed(seed)
    B, (ih, iw) = g.B, g.in_hw
    fr = [(R.smooth(B, ih, iw, 3, 0.3, gen) + 0.2 * (torch.rand(B, ih, iw, 3, generator=gen) - 0.5)).clamp(-0.5, 0.5) for _ in range(2)]
    gt = R.smooth(B, ih, iw, 2, 4.0, gen, div=24)
    g.img1.copy_(fr[0])
    g.img2.copy_(fr[1])
    g.gt.copy_(gt)


# ------------------------------------------------------------------------------------------------ poisoned replay
def _targets(g):
    """Acts and fp32 / fp64 tensors the plans of g write (inputs, parameters, m, v, step and lr excluded)."""
    keep = {t.untyped_storage().data_ptr() for t in (g.store.flat, g.store.m, g.store.v, g.store.grad, g.step_state, g.lr) + tuple(g.inputs)}
    acts, f32, seen = [], [], set()

    def walk(o):
        if o is None or id(o) in seen:
            return
        seen.add(id(o))
        if isinstance(o, E.Act):
            acts.append(o)
            walk(o.grad)
        elif isinstance(o, torch.Tensor):
            if o.dtype in (torch.float32, torch.float64) and o.is_cuda and o.untyped_storage().data_ptr() not in keep:
                f32.append(o)
        elif isinstance(o, (list, tuple)):
            for x in o:
                walk(x)
        elif isinstance(o, dict):
            for x in o.values():
                walk(x)
        elif isinstance(o, E.ConvLayer):
            for x in (o.dcat, o.dwp, o.colpart, o.dwp_hi):
                walk(x)
            for pk in o.tr_packs or ():
                walk(pk.dwp)
            if o.tr_planes is not None:
                f32.append(o.tr_planes)
    walk(g.bld.keep)
    for _, p in ((n, getattr(g, n)) for n in PLANS):
        walk(p.keep)
    for L in g.pwc.all_layers():
        walk(L)
    named = [g.flow, g.sums, g._scratch] + ([g.aug_params] + list(g.batch) if g.augment else [])
    named += [getattr(g, k) for k in ('warped', 'mask', 'coef', 'dflow') if hasattr(g, k)]
    f32 += [t for t in named if all(t is not x for x in f32)]
    return acts, f32


def _poison(g, sentinel):
    acts, f32 = _targets(g)
    for a in acts:
        idx = [a.c_off + p for p, m in enumerate(a.chanmap) if m >= 0]
        if not idx:
            continue
        v = torch.full((a.N, a.H, a.W, len(idx)), sentinel, dtype=torch.bfloat16, device='cuda')
        if sentinel == sentinel:
            v[..., 1::2] = -sentinel
        a.buf[:a.N].index_copy_(3, torch.tensor(idx, device='cuda'), v)
    for t in f32:
        t.fill_(sentinel)
        if sentinel == sentinel:
            t.view(-1)[1::2] = -sentinel
    st = g.store
    for name, _, n, off, _ in st.entries:
        st.grad[off:off + n].fill_(sentinel)


def _bits(t):
    return t.view(torch.int32 if t.element_size() == 4 else torch.int64)


def _poisoned_replays(g, clean):
    """Capture fwd_bwd (warm run, then capture), poison, replay -> {sentinel: (poisoned, identical)}."""
    out = {}
    graph = g._capture('fwd_bwd', [g.aug, g.fwd, g.bwd])
    for sentinel in (float('nan'), 2.0 ** 100):
        _poison(g, sentinel)
        torch.cuda.synchronize()
        poisoned = not torch.equal(_bits(g.store.grad), _bits(clean['grad']))
        graph.replay()
        torch.cuda.synchronize()
        out[sentinel] = (poisoned, all(torch.equal(_bits(getattr(g.store, 'grad') if k == 'grad' else g.sums), _bits(v))
                                       for k, v in clean.items()))
    return out


# ------------------------------------------------------------------------------------------------ the walk
def _pack_check(g, glue):
    """Unsupervised graph: the image Acts hold bf16(frame + 0.5) of (frame 1, frame 2) and (frame 2, frame 1); the control takes the
    second half of each from the other frame."""
    B = g.B
    fr = [G.decode(op)['dst'] for op in g.fwd.ops if op[2] == 'cis_resize_bilinear_f32'][:2]
    fr = [glue.mem.view(p, torch.float32, (B, g.H, g.W, 3)) for p in fr]
    want = [(fr[0], fr[1]), (fr[1], fr[0])]
    r, bad = 0.0, 0.0
    for a, (first, second) in zip(g.img_acts, want):
        got = a.buf[:2 * B, ..., :3]
        ref = torch.cat([first, second]) + torch.tensor(0.5, dtype=torch.float32)
        r = max(r, G.exact(got, ref))
        bad = max(bad, G.exact(got, torch.cat([first, first]) + torch.tensor(0.5, dtype=torch.float32)))
    return r, bad


def _epe_check(g):
    """epe() after the walked forward against fp64: the legacy-bilinear resize of the prediction to the ground truth's grid with its
    vectors scaled by (ih / H, iw / W), then per-sample sums of ||pred - gt||.  Bound: the resize's 2^-21 sum |corners| |scale| per
    channel (1-Lipschitz norm), plus the fp64 sums."""
    (ih, iw), H, W, B = g.in_hw, g.H, g.W, g.B
    got = g.epe().clone()
    torch.cuda.synchronize()
    f = g.flow.double()
    gt = g.batch[2].double()
    (My, Iy), (Mx, Ix) = G.lerp_axis(H, ih), G.lerp_axis(W, iw)
    sc = torch.tensor([float(G._f32(ih / H)), float(G._f32(iw / W))], dtype=torch.float64, device='cuda')
    pred = G.apply2(My, Mx, f) * sc
    e = (G.G_LERP * G.apply2(Iy, Ix, f.abs()) * sc).sum(-1)
    epe = torch.sqrt(((pred - gt) ** 2).sum(-1))
    ref = torch.stack([epe.sum((1, 2)), torch.zeros(B, dtype=torch.float64, device='cuda'),
                       torch.full((B,), float(ih * iw), dtype=torch.float64, device='cuda'), torch.zeros(B, dtype=torch.float64, device='cuda')], 1)
    b = torch.stack([e.sum((1, 2)) + (ih * iw + 128) * 2.0 ** -53 * epe.sum((1, 2)), torch.zeros(B, dtype=torch.float64, device='cuda'),
                     torch.zeros(B, dtype=torch.float64, device='cuda'), torch.zeros(B, dtype=torch.float64, device='cuda')], 1)
    return G.ratio(got, ref, b)


def _walk_step(g, rec, step, out, poison=False):
    glue = G.Glue(controls=True)
    w = R.Walker(rec, controls=True, glue=glue)
    counts = {}
    for name in PLANS:
        plan = getattr(g, name)
        n, m = len(w.failures), len(glue.failures)
        before = dict(glue.counts)
        w.run(plan)
        counts[name] = {k: v - before.get(k, 0) for k, v in glue.counts.items() if v - before.get(k, 0)}
        out['failures'] += ['step %d %s: %s' % (step, name, f) for f in w.failures[n:] + glue.failures[m:]]
        if name == 'fwd' and g.loss == 'unsupervised':
            r, bad = _pack_check(g, glue)
            out['pack'] = max(out.get('pack', 0.0), r)
            glue._control('pack.unswapped', bad)
        if name == 'fwd' and step == 1 and GRAPHS_EPE.get(out['key']):
            out['epe'] = _epe_check(g)
        if name == 'bwd' and poison:
            torch.cuda.synchronize()
            out['poison'] = _poisoned_replays(g, dict(grad=g.store.grad.clone(), sums=g.sums.clone()))
    out['counts'].append(counts)
    out['conv'].append(w.checked)
    for k, v in dict(w.controls, **glue.controls).items():
        out['controls'][k] = max(out['controls'].get(k, 0.0), v) if k not in UNREJECTED else v
    for lab, v in list(w.summary().items()) + list(glue.summary().items()):
        print('%-8s step %d %-44s count %4d  worst bound ratio %.3g' % (out['key'], step, lab, v['count'], v['worst']))
        out['worst'][lab] = max(out['worst'].get(lab, 0.0), v['worst'])
    if hasattr(glue, 'unsup_mask'):
        print('%-8s step %d unsupervised mask vs fp64: %s' % (out['key'], step, glue.unsup_mask))


GRAPHS_EPE = {'default': True}
_WALKS = {}


def walk(key):
    if key in _WALKS:
        return _WALKS[key]
    t0 = time.time()
    g, rec, _ = build(key, 'cuda')
    opts = GRAPHS[key][1].get('options')
    g.load_params(REF.make_params(3, jitter=0.1, options=opts))
    _inputs(g, 40 + KEYS.index(key))
    g._ensure_packed()
    out = dict(key=key, failures=[], counts=[], conv=[], controls={}, worst={}, tables=[])
    for step in (1, 2):
        _walk_step(g, rec, step, out, poison=step == 1)
        if g.augment:
            out['tables'].append(g.aug_params.clone())
    out['step_state'] = int(g.step_state)
    print('%-8s negative controls (ratio > 1 = rejected): %s' % (key, out['controls']))
    print('%-8s %s conv and %s glue launches checked over two steps in %.1f s'
          % (key, out['conv'], [sum(sum(c.values()) for c in s.values()) for s in out['counts']], time.time() - t0))
    del g, rec
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    _WALKS[key] = out
    return out


@pytest.mark.parametrize('key', KEYS)
def test_every_launch_within_its_bound(key):
    r = walk(key)
    assert not r['failures'], '%s:\n%s' % (key, '\n'.join(r['failures'][:20]))
    assert r['conv'] == [CONV[key]] * 2
    assert r['counts'] == [GLUE[key]] * 2, r['counts']
    assert r['step_state'] == 2
    if key == 'unsup':
        assert r['pack'] == 0.0


@pytest.mark.parametrize('key', KEYS)
def test_negative_controls_are_rejected(key):
    c = walk(key)['controls']
    want = {'tile', 'fwd.halo', 'adam.decay_everywhere', 'adam.t_off_by_one'}
    if key == 'unsup':
        want |= {'unsup.mask_ones', 'unsup_bwd.smooth_dropped', 'pack.unswapped'}
    else:
        want |= {'ms_loss.level_scale', 'ms_loss_bwd.weights_reversed', 'tile.cis_flow_multiscale_loss_bwd'}
    if key in ('default', 'shard'):
        want |= {'ms_loss.axes_swapped'}
    if key == 'shard':
        want |= {'aug_params.step_frozen', 'augment.flow_unmapped'}
    assert want <= set(c), (key, sorted(want - set(c)))
    bad = {k: v for k, v in c.items() if k not in UNREJECTED and not v > 1.0}
    assert not bad, (key, bad)


@pytest.mark.parametrize('key', KEYS)
def test_poisoned_graph_replay_is_bit_identical(key):
    for sentinel, (poisoned, same) in walk(key)['poison'].items():
        assert poisoned and same, (key, sentinel, poisoned, same)


def test_augmentation_redraws_at_step_two():
    t = walk('shard')['tables']
    assert len(t) == 2 and not torch.equal(t[0], t[1])


def test_default_epe_matches_fp64():
    r = walk('default')['epe']
    print('default epe() vs fp64: worst bound ratio %.3g' % r)
    assert r <= 1.0


def test_unsup_loss_launches_on_partly_consistent_flows():
    """The untrained network's two directions disagree almost everywhere, so in the `unsup` walk the mask keeps few pixels.  Here the
    same two launches run on flows built to be partly consistent (the backward flow is minus the forward one plus a smooth field, as in
    tests/test_unsup_flow_gpu.py), so that the census, coef and gather references are compared on many visible pixels."""
    gen = torch.Generator().manual_seed(77)
    B, H, W = 2, 192, 384
    N = 2 * B
    fr = [(R.smooth(B, H, W, 3, 0.3, gen) + 0.2 * (torch.rand(B, H, W, 3, generator=gen) - 0.5)).clamp(-0.5, 0.5).cuda() for _ in range(2)]
    ff = R.smooth(B, H, W, 2, 3.0, gen)
    flow = torch.cat([ff, -ff + R.smooth(B, H, W, 2, 1.0, gen)]).contiguous().cuda()
    warped, mask, coef = (torch.full((N, H, W), float('nan'), device='cuda') for _ in range(3))
    scratch = torch.full((2 * N * 64,), float('nan'), dtype=torch.float64, device='cuda')
    out = torch.full((N, 2), float('nan'), dtype=torch.float64, device='cuda')
    dflow = torch.full((N, H, W, 2), float('nan'), device='cuda')
    ptrs = (flow.data_ptr(), fr[0].data_ptr(), fr[1].data_ptr(), B, H, W)
    plan = E.Plan('direct_unsup')
    plan.add('cis_unsup_flow_loss', *ptrs, warped.data_ptr(), mask.data_ptr(), coef.data_ptr(), scratch.data_ptr(), out.data_ptr())
    norm = float(4 * H * W)
    plan.add('cis_unsup_flow_loss_bwd', *ptrs, warped.data_ptr(), coef.data_ptr(), 1.0 / norm, 3.0 / norm, dflow.data_ptr())
    glue = G.Glue(controls=True)
    R.Walker(R.Recorder(), glue=glue).run(plan)
    for lab, v in glue.summary().items():
        print('direct_unsup %-40s count %4d  worst bound ratio %.3g' % (lab, v['count'], v['worst']))
    print('direct_unsup mask vs fp64: %s; controls %s' % (glue.unsup_mask, glue.controls))
    assert not glue.failures, '\n'.join(glue.failures[:20])
    assert dict(glue.counts) == {'cis_unsup_flow_loss': 1, 'cis_unsup_flow_loss_bwd': 1}
    m = glue.unsup_mask
    assert m['pixels'] - m['out'] - m['occluded'] >= 0.1 * m['pixels'] and m['out'] > 0 and m['occluded'] > 0, m
    assert glue.controls['unsup.mask_ones'] > 1.0 and glue.controls['unsup_bwd.smooth_dropped'] > 1.0, glue.controls


def test_abs_sum_matches_fp64():
    """cis_abs_sum: stat[0] += sum |g| (fp32 lanes over a grid-stride loop, a warp sum, atomic adds of 296 * 8 warp partials)."""
    gen = torch.Generator().manual_seed(9)
    n = 1000003
    g = (torch.randn(n, generator=gen) * torch.rand(n, generator=gen) ** 4).cuda()
    stat = torch.tensor([0.25], device='cuda')
    _lib.call('cis_abs_sum', g.data_ptr(), n, stat.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    ref = 0.25 + g.double().abs().sum()
    terms = -(-n // (296 * 256)) + 5 + 296 * 8 + 1
    assert abs(float(stat) - float(ref)) <= terms * G.U23 * float(ref)
