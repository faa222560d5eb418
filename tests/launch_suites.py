"""The harness of the per-launch check suites (tests/test_*launches*_{cpu,gpu}.py) around the two checkers, tests/conv_launch_ref.py and
tests/glue_launch_ref.py.

  GRAPHS        the registry: each key names one graph that also builds on CPU tensors, with its constructor, its [(plan name, Plan)]
                list and its seeded parameters and inputs.  The CPU files build them without launching anything and pin their census
                (CONV, GLUE); the GPU files walk them.
  walk_plans    one replay of a list of plans with both checkers, Walker(rec, glue=Glue()): per-plan failures and glue counts, conv
                launches checked, the merged negative controls and one summary line per launch label.
  walk_graph    the checked replay of a registry graph on the GPU, made once per test session and shared by every test that asserts on it.
  report        prints a summary and the controls (pytest -s shows them).
  targets, poison, bits
                the poisoned-buffer replays: every buffer a graph's plans write is filled with NaN, then with +-2^100, and the replay must
                leave its outputs bit-identical.
"""
import collections
import functools
import time

import pytest
import torch

import conv_launch_ref as R
import glue_launch_ref as G
import pwc_options_ref as REF
from oracle import params as OP
from unsupervised_detection_b200 import engine as E
from unsupervised_detection_b200.flow_train_graph import FlowTrainGraph
from unsupervised_detection_b200.models import functional as FN
from unsupervised_detection_b200.models.PWCNet.model_pwcnet import _DEFAULT_PWCNET_TEST_OPTIONS
from unsupervised_detection_b200.step_graph import CISGraph

# Controls the bound is not expected to reject in a graph walk: the leaky gate of the warp + cost-volume transpose hardly shows where the
# pyramid's correlations are almost all positive (test_glue_launches_gpu.py checks it on independent random features).
UNREJECTED = {'costvol_bwd.gate_one'}


# ------------------------------------------------------------------------------------------------------------ census tables
# glue launches per plan
CONFIG2 = {
    'fwd': {'cis_resize_concat_bf16': 11, 'cis_warp_costvol': 5, 'cis_pack_f32_to_bf16': 3, 'cis_resize_bilinear_f32': 3,
            'cis_upsample_nn2x': 2, 'cis_flow_stats': 1, 'cis_pack_generator_input': 1, 'cis_zero': 2},
    'bwd_R': {'cis_dact_colsum': 23, 'cis_resize_concat_bf16_bwd': 14, 'cis_colsum': 9},
    'bwd_G': {'cis_dact_colsum': 16, 'cis_dact_mul': 14, 'cis_resize_concat_bf16_bwd': 14, 'cis_add_slice': 3, 'cis_upsample_nn2x_bwd': 2,
              'cis_colsum': 1},
}
PWC_BWD = {'cis_dact_colsum': 91, 'cis_colsum': 18, 'cis_parity_split_bf16': 8, 'cis_warp_costvol_bwd': 5, 'cis_zero': 5,
           'cis_cast_bf16_to_f32': 2, 'cis_resize_f32_bwd_to_bf16_scaled': 1}
PWC_FWD = {'cis_warp_costvol': 5, 'cis_pack_f32_to_bf16': 2, 'cis_resize_bilinear_f32': 1}
# the flow given directly: no PWC-Net, no 384x640 inputs
FLOW_GIVEN = dict(CONFIG2, fwd={'cis_resize_concat_bf16': 11, 'cis_pack_f32_to_bf16': 1, 'cis_upsample_nn2x': 2, 'cis_flow_stats': 1,
                                'cis_pack_generator_input': 1, 'cis_zero': 2})
BOXES = {'fwd': {'cis_resize_concat_bf16': 11, 'cis_warp_costvol': 5, 'cis_pack_f32_to_bf16': 3, 'cis_resize_bilinear_f32': 3, 'cis_zero': 1},
         'bwd_R': CONFIG2['bwd_R']}
# the inference graphs: 'masks' = _mask_plan, 'rest' = the other forward ops
GEN_FWD = {'masks': {'cis_zero': 1, 'cis_flow_stats': 1, 'cis_pack_generator_input': 1, 'cis_pack_f32_to_bf16': 1, 'cis_upsample_nn2x': 2},
           'rest': {'cis_resize_concat_bf16': 11, 'cis_zero': 1}}
ENSEMBLE = {'masks': {'cis_pack_f32_to_bf16': 3, 'cis_warp_costvol': 5, 'cis_resize_bilinear_f32': 3, 'cis_zero': 1, 'cis_flow_stats': 1,
                      'cis_pack_generator_input': 1, 'cis_upsample_nn2x': 2},
            'rest': {'cis_resize_concat_bf16': 11, 'cis_zero': 1}}
# search ranges 1-3: the warp + cost-volume launches take the entry points with a range argument
PWC_RANGE = {plan: {n + '_r' if n.startswith('cis_warp_costvol') else n: c for n, c in counts.items()}
             for plan, counts in (('fwd', PWC_FWD), ('bwd', PWC_BWD))}
# the PWC-Net training step
TRAIN_BWD = {'cis_zero': 5, 'cis_flow_multiscale_loss_bwd': 1, 'cis_colsum': 18, 'cis_dact_colsum': 91, 'cis_warp_costvol_bwd': 5,
             'cis_parity_split_bf16': 8}
TRAIN_FWD = {'cis_resize_bilinear_f32': 3, 'cis_pack_f32_to_bf16': 2, 'cis_warp_costvol': 5, 'cis_flow_multiscale_loss': 1}
TRAIN_DEFAULT = {'aug': {}, 'fwd': TRAIN_FWD, 'bwd': TRAIN_BWD, 'adam': {'cis_adam_l2': 1}, 'pack': {}}
GLUE = {
    'config2': CONFIG2, 'boxes': BOXES, 'defaults': FLOW_GIVEN, 'odd': FLOW_GIVEN, 'gen_fwd': GEN_FWD, 'ensemble': ENSEMBLE,
    'pwc_runner': {'fwd': PWC_FWD, 'bwd': PWC_BWD}, 'r1': PWC_RANGE, 'r2': PWC_RANGE, 'r3': PWC_RANGE,
    'dense_off': {'fwd': PWC_FWD, 'bwd': PWC_BWD},
    'default': TRAIN_DEFAULT,
    'unsup': dict(TRAIN_DEFAULT,
                  fwd={'cis_resize_bilinear_f32': 3, 'cis_pack_f32_to_bf16': 4, 'cis_warp_costvol': 5, 'cis_unsup_flow_loss': 1},
                  bwd=dict({k: v for k, v in TRAIN_BWD.items() if k != 'cis_flow_multiscale_loss_bwd'}, cis_unsup_flow_loss_bwd=1,
                           cis_resize_f32_bwd_to_bf16_scaled=1)),
    'timed': dict(TRAIN_DEFAULT, fwd=dict(TRAIN_FWD, cis_resize_bilinear_f32=1)),     # no input resize: only the final x4
    'shard': dict(TRAIN_DEFAULT, aug={'cis_flow_aug_params': 1, 'cis_flow_augment': 1}),
}
# conv launches per graph (cis_conv_igemm + cis_conv_wgrad ops over its plans; the PWC-Net training step: fwd + bwd)
CONV = {'gen_fwd': 49, 'ensemble': 158, 'odd': 185, 'r1': 357, 'r2': 357, 'r3': 357, 'dense_off': 357,
        'default': 367, 'unsup': 367, 'timed': 355, 'shard': 367}


# ------------------------------------------------------------------------------------------------------------ seeded inputs
def frames(B, H, W, seed):
    """A smooth frame in [-0.5, 0.5] and the same frame rolled by (2, 3) pixels plus 0.01 noise, and the generator for what follows."""
    gen = torch.Generator().manual_seed(seed)
    img1 = R.smooth(B, H, W, 3, 0.25, gen).clamp(-0.5, 0.5)
    return img1, torch.roll(img1, shifts=(2, 3), dims=(1, 2)) + 0.01 * torch.randn(B, H, W, 3, generator=gen), gen


def _with_pwc(g):
    """Every network, frames of seed 7 at PWC-Net's input size."""
    g.load_params(OP.make_params(seed=1, jitter=0.1))
    img1, img2, _ = frames(*g.img1.shape[:3], 7)
    g.img1.copy_(img1)
    g.img2.copy_(img2)
    g._ensure_packed()


def _flow_given(seed):
    """The generator and recover nets, a random image and a smooth flow."""
    def inputs(g):
        g.load_params(OP.make_params(seed=4, jitter=0.1, nets=('MaskNet', 'FlownetS')))
        gen = torch.Generator().manual_seed(seed)
        g.image.copy_(torch.rand(g.B, g.H, g.W, 3, generator=gen) - 0.5)
        g.flow.copy_(R.smooth(g.B, g.H, g.W, 2, 0.3, gen))
        g._ensure_packed()
    return inputs


def _pwc_runner(params):
    """Frames of seed 13 and a smooth flow gradient to propagate back."""
    def inputs(r):
        r.reload(params())
        img1, img2, gen = frames(r.B, r.H, r.W, 13)
        r.img1.copy_(img1)
        r.img2.copy_(img2)
        r.dflow_out.copy_(R.smooth(r.B, r.H, r.W, 2, 1.0, gen))
    return inputs


def _flow_train(seed, options=None):
    """Textured frames in [-0.5, 0.5] (tests/test_unsup_flow_gpu.py's construction) and a smooth ground truth of several pixels, at the
    upload size."""
    def inputs(g):
        g.load_params(REF.make_params(3, jitter=0.1, options=options))
        gen = torch.Generator().manual_seed(seed)
        B, (ih, iw) = g.B, g.in_hw
        fr = [(R.smooth(B, ih, iw, 3, 0.3, gen) + 0.2 * (torch.rand(B, ih, iw, 3, generator=gen) - 0.5)).clamp(-0.5, 0.5) for _ in range(2)]
        g.img1.copy_(fr[0])
        g.img2.copy_(fr[1])
        g.gt.copy_(R.smooth(B, ih, iw, 2, 4.0, gen, div=24))
        g._ensure_packed()
    return inputs


# ------------------------------------------------------------------------------------------------------------ the registry
def _cis_plans(g):
    return [('fwd', g.fwd)] + [('bwd_' + m, p) for m, p in g.bwd.items()]


def split_fwd(g):
    """[('masks', _mask_plan), ('rest', the forward ops that are not in it, in plan order)].  Ops are matched by identity, counted: the
    structural 'join' op is one shared tuple that can appear in both parts."""
    left = collections.Counter(id(op) for op in g._mask_plan.ops)
    rest = E.Plan('fwd_rest')
    for op in g.fwd.ops:
        if left[id(op)]:
            left[id(op)] -= 1
        else:
            rest.ops.append(op)
    assert not +left
    rest.keep = g.fwd.keep
    return [('masks', g._mask_plan), ('rest', rest)]


def _cis(*a, **kw):
    return lambda device: CISGraph(*a, device=device, **kw)


def _pwc(options=None):
    def make(device):
        r = FN._PWCRunner(2, 384, 640, device, 'pwcnet', trainable=True, options=options)
        r.ensure_backward()
        return r
    return make


def _pwc_plans(r):
    return [('fwd', r.bld.fwd), ('bwd', r.bwd)]


PLANS = ('aug', 'fwd', 'bwd', 'adam', 'pack')


def _train(*a, **kw):
    return lambda device: FlowTrainGraph(*a, device=device, **kw)


def _train_plans(g):
    return [(p, getattr(g, p)) for p in PLANS]


PWC_OPTIONS = {'r1': {'search_range': 1}, 'r2': {'search_range': 2}, 'r3': {'search_range': 3}, 'dense_off': {'use_dense_cx': False}}
_SHARD = dict(global_batch=16, in_hw=(384, 640), loss='robust', options={'use_dense_cx': False}, augment=True, sample_offset=8)

# key -> (constructor(device), [(plan name, Plan)] of the graph, parameters and inputs of the graph on the GPU)
GRAPHS = {
    # the train step at 256x448, batch 4, PWC-Net at 384x640 (bench.py's config 2), and with box-shaped masks
    'config2': (_cis(256, 448, 4, with_pwc=True, train=True), _cis_plans, _with_pwc),
    'boxes': (_cis(256, 448, 4, with_pwc=True, train=True, masks='boxes'), _cis_plans, _with_pwc),
    # the reference's default geometry (common_flags.py), and a size that is not a multiple of 64, with the flow given directly
    'defaults': (_cis(192, 384, 16, with_pwc=False, train=True), _cis_plans, _flow_given(3)),
    'odd': (_cis(100, 172, 3, with_pwc=False, train=True), _cis_plans, _flow_given(5)),
    # the inference graphs of bench.py --workload gen_fwd / ensemble: the mask plan, then the rest of the forward
    'gen_fwd': (_cis(128, 224, 1, with_pwc=False, train=False), split_fwd, _flow_given(5)),
    'ensemble': (_cis(192, 384, 4, train=False, pwc_options=_DEFAULT_PWCNET_TEST_OPTIONS), split_fwd, _with_pwc),
    # PWC-Net forward and backward at 384x640, batch 2: the default options, search ranges 1-3, no dense connections
    'pwc_runner': (_pwc(), _pwc_plans, _pwc_runner(lambda: OP.make_params(seed=1, jitter=0.1))),
    **{k: (_pwc(o), _pwc_plans, _pwc_runner(functools.partial(REF.make_params, 1, jitter=0.1, options=o))) for k, o in PWC_OPTIONS.items()},
    # the PWC-Net training step: train_flow.py's defaults on one GPU, the unsupervised loss, tools/time_flow_train.py's timed step, and
    # rank 2 of 4 with the robust loss, the "sm" network and the augmentation
    'default': (_train(192, 384, 16, in_hw=(384, 640)), _train_plans, _flow_train(40)),
    'unsup': (_train(192, 384, 16, in_hw=(384, 640), loss='unsupervised'), _train_plans, _flow_train(41)),
    'timed': (_train(384, 640, 8), _train_plans, _flow_train(42)),
    'shard': (_train(192, 384, 4, **_SHARD), _train_plans, _flow_train(43, _SHARD['options'])),
}
VARIANTS = ['gen_fwd', 'ensemble', 'odd'] + list(PWC_OPTIONS)
FLOW_TRAIN = ['default', 'unsup', 'timed', 'shard']


def build(key, device):
    """(graph, conv Recorder, [(plan name, Plan)]) of registry key `key`."""
    make, plans, _ = GRAPHS[key]
    with R.recorded(pytest.MonkeyPatch()) as rec:
        g = make(device)
    return g, rec, plans(g)


def load_inputs(key, g):
    GRAPHS[key][2](g)


# ------------------------------------------------------------------------------------------------------------ conv-op attribution
def attributed(rec, plans):
    """Every conv op of `plans` maps to one check, every op of such a check is in the same plan, in order, each op in one check only."""
    seen = collections.Counter()
    checks = []
    for plan in plans:
        pos = {id(op): i for i, op in enumerate(plan.ops)}
        for op in R.conv_ops(plan):
            ck = rec.by_op.get(id(op))
            assert ck is not None, ('unattributed', op[2], plan.name)
            seen[id(op)] += 1
            if ck.ops[0] is op:
                idx = [pos.get(id(o)) for o in ck.ops]
                assert None not in idx and idx == sorted(idx), ck
                checks.append(ck)
    assert all(v == 1 for v in seen.values())
    return checks


def features(checks):
    """The launch configurations `checks` reach, for the coverage tests."""
    f = set()
    for ck in checks:
        for d in ck.descs():
            if ck.kind == 'wgrad':
                f.add(('wgrad.tma', d.tma))
                f.add(('wgrad.nwg', d.nwg))
                f.add(('wgrad.split', d.splits > 1))
                if d.tma == 2:
                    f.add(('wgrad.nh', d.nh))
                if any(b.data_ptr() <= d.dwp < b.data_ptr() + 4 * b.numel() for b in ck.layer.dwp_hi.values()):
                    f.add('wgrad.cout_hi')
                continue
            if ck.kind == 'dgrad' and d.nsub == 4 and d.add_pre:
                f.add(('dgrad.nsub4_add_pre.BN', d.BN))
            if ck.kind == 'dgrad' and d.n_tiles >= 3:
                f.add('dgrad.n_tiles>=3')
            if d.halo and d.splits > 2:
                f.add('halo.splits>2')
            if not d.halo and d.splits > 1:
                f.add('gather.splitk')
            if d.nwg == 2:
                f.add('nwg2')
                if d.add_post:
                    f.add('add_post.nwg2')
            if d.halo and d.dil > 1:
                f.add(('dil', d.dil))
            if any(d.src[i].n_mod for i in range(d.nsrc)):
                f.add(('n_mod', d.nsrc, max(d.splits, 1)))
            if d.addf_pre:
                f.add('addf_pre' + ('.outf' if d.outf else ''))
            if d.add_post:
                f.add('add_post')
            if d.mode == 1:
                f.add('mode1')
            if d.nsub > 1 and d.outf:
                f.add('parity_group.outf')
    return f


# ------------------------------------------------------------------------------------------------------------ the walk
def walk_plans(rec, plans, controls=False, glue_controls=False, after=None):
    """One replay of `plans` ([(name, Plan)]) with every conv launch `rec` recorded and every glue launch checked, after(name, glue) called
    after each plan -> dict(failures={plan: [message]}, counts={plan: {entry point: glue launches}}, conv=conv launches checked,
    glue=glue launches checked, controls=both checkers' negative controls (None when neither made any), summary={label: dict(count,
    worst[, persist])}, unsup_mask, first_nonfinite)."""
    glue = G.Glue(controls=glue_controls)
    w = R.Walker(rec, controls=controls, glue=glue)
    failures, counts = {}, {}
    for name, plan in plans:
        n, m, before = len(w.failures), len(glue.failures), dict(glue.counts)
        w.run(plan)
        failures[name] = w.failures[n:] + glue.failures[m:]
        counts[name] = {k: v - before.get(k, 0) for k, v in glue.counts.items() if v - before.get(k, 0)}
        if after is not None:
            after(name, glue)
    cand = R.count_persist(rec, [p for _, p in plans])
    summary = {lab: dict(v, persist=cand[lab][1] if lab in cand else 0) for lab, v in w.summary().items()}
    summary.update(glue.summary())
    controls = None
    if w.controls is not None or glue.controls is not None:
        controls = dict(w.controls or {}, **(glue.controls or {}))
    return dict(failures=failures, counts=counts, conv=w.checked, glue=sum(glue.counts.values()), controls=controls, summary=summary,
                unsup_mask=getattr(glue, 'unsup_mask', None), first_nonfinite=glue.first_nonfinite)


def assert_within_bounds(r, *plans):
    """No launch of `plans` (all of them by default) of walk result `r` failed; the first 20 that did are named."""
    bad = ['%s: %s' % (p, f) for p in plans or r['failures'] for f in r['failures'][p]]
    assert not bad, '\n'.join(bad[:20])


def report(key, summary, controls=None):
    """One line per launch label: count, worst bound ratio and, for a conv label, the descriptor-side candidates of the persistent
    kernel; then the controls."""
    for lab, v in summary.items():
        cand = '  persistent-kernel candidates %d' % v['persist'] if 'persist' in v else ''
        print('%-22s %-44s count %4d  worst bound ratio %.3g%s' % (key, lab, v['count'], v['worst'], cand))
    if controls is not None:
        print('%-22s negative controls (ratio > 1 = rejected): %s' % (key, controls))


# The defaults graph is walked without negative controls and the PWC runner with the glue ones only: config 2, odd and the PWC-Net
# variants make every control of those launch kinds.  Every other graph: both checkers' controls.
_CONTROLS = {'defaults': (False, False), 'pwc_runner': (False, True)}


@functools.lru_cache(maxsize=None)
def walk_graph(key):
    """The checked replay of registry graph `key` (a CISGraph or a PWC runner) on the GPU -> walk_plans' result plus bn_fold (the worst
    ratio of the generator's folded BN weights, 0 without a generator) and, for a graph with a mask plan, mask (what the replay of that plan
    left) and graph_mask {sentinel: (whether poisoning changed the mask, the mask a replay of the captured forward_masks graph then
    left)}.  Made once per session; the graph and its buffers are released."""
    t0 = time.time()
    g, rec, plans = build(key, 'cuda')
    load_inputs(key, g)
    masks = {}

    def after(name, glue):
        if name == 'masks':
            masks['walk'] = g.mask.clone()

    out = walk_plans(rec, plans, *_CONTROLS.get(key, (True, True)), after=after)
    out.update(bn_fold=R.check_bn_fold(g.gen.all_layers()) if isinstance(g, CISGraph) else 0.0, mask=masks.get('walk'), graph_mask=None)
    if masks:
        # The first call captures the CUDA graph (after running the plan eagerly once); every buffer the plans write is then poisoned
        # and the second call only replays the graph, so the mask it leaves is the captured graph's own work.
        g.forward_masks(use_graph=True)
        out['graph_mask'] = {}
        for sentinel in (float('nan'), 2.0 ** 100):
            poison_cis(g, [], sentinel)
            torch.cuda.synchronize()
            poisoned = not torch.equal(g.mask, out['mask'])
            assert set(g.graphs) == {'masks'}
            g.forward_masks(use_graph=True)
            torch.cuda.synchronize()
            out['graph_mask'][sentinel] = (poisoned, g.mask.clone())
    report(key, out['summary'], out['controls'])
    print('%-22s %d conv and %d other launches checked in %.1f s' % (key, out['conv'], out['glue'], time.time() - t0))
    del g, rec, plans
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return out


# ------------------------------------------------------------------------------------------------------------ poisoned replays
def targets(roots, named, excluded):
    """(Acts, other tensors) for poison(): the `named` buffers, then every Act and fp32 / fp64 CUDA tensor reachable from `roots` (plan
    keep lists, ConvLayers: their dcat, weight-gradient slices, partial sums and bf16 parity planes) that does not start where a named one
    does; none that shares storage with one of `excluded` (what a batch upload writes, parameters)."""
    skip = {t.untyped_storage().data_ptr() for t in excluded}
    acts, found, seen = [], [], set()

    def walk(o):
        if o is None or id(o) in seen:
            return
        seen.add(id(o))
        if isinstance(o, E.Act):
            acts.append(o)
            walk(o.grad)
        elif isinstance(o, torch.Tensor):
            if o.dtype in (torch.float32, torch.float64) and o.is_cuda and o.untyped_storage().data_ptr() not in skip:
                found.append(o)
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
                found.append(o.tr_planes)
    walk(roots)
    named = [t for t in named if t.untyped_storage().data_ptr() not in skip]
    starts = {t.data_ptr() for t in named}
    return acts, named + [t for t in found if t.data_ptr() not in starts]


def poison(found, stores, sentinel):
    """Fill the real channels of the Acts and the tensors targets() found, and the real entries of the flat gradients of `stores`, with
    `sentinel` (a finite one alternating in sign)."""
    acts, tensors = found
    for a in acts:
        idx = [a.c_off + p for p, m in enumerate(a.chanmap) if m >= 0]
        if not idx:
            continue
        v = torch.full((a.N, a.H, a.W, len(idx)), sentinel, dtype=torch.bfloat16, device='cuda')
        if sentinel == sentinel:
            v[..., 1::2] = -sentinel
        a.buf[:a.N].index_copy_(3, torch.tensor(idx, device='cuda'), v)
    for t in tensors:
        t.fill_(sentinel)
        if sentinel == sentinel:
            t.view(-1)[1::2] = -sentinel
    for st in stores:
        for name, _, n, off, _ in st.entries:
            st.grad[off:off + n].fill_(sentinel)


def poison_cis(g, modes, sentinel):
    """Poison what the fwd plan and the bwd plans of `modes` of CISGraph `g` write, and the flat gradients of those modes."""
    plans = [g.fwd] + [g.bwd[m] for m in modes]
    layers = list(g.gen.all_layers()) + list(g.rec.all_layers()) + (list(g.pwc.all_layers()) if g.with_pwc else [])
    # scalars[5:8] are slots no kernel writes (cis_cis_loss_reduce defines [0, 5))
    named = [g.image, g.flow, g.mask, g.flow1, g.pred, g.dmask, g.sums, g.scalars[:5], g.coef]
    named += [t for t in (getattr(g, 'dpred', None), getattr(g, 'stats', None), getattr(g, 'image_st', None), getattr(g, 'flow_st', None))
              if t is not None]
    if g.with_pwc:
        named.append(g.flow_full)
    # what a batch upload writes (the two buffers of a staged graph, image and flow otherwise) is input, not poisoned
    found = targets([g.bld.keep] + [p.keep for p in plans] + layers, named, g.inputs if g.staged else (g.image, g.flow))
    poison(found, [g.store(m) for m in modes], sentinel)


def bits(t):
    return t.view(torch.int32 if t.element_size() == 4 else torch.int64)
