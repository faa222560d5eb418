"""Every launch of the graphs the project ships besides the three of tests/test_conv_launches_gpu.py, checked on its own against an fp64
reference: the conv launches by tests/conv_launch_ref.py, the others by tests/glue_launch_ref.py, in one replay per plan
(Walker(rec, glue=Glue())), with every negative control of both checkers.  The graphs and why each one
(tests/test_graph_variants_launches_cpu.py pins their launch census):

  gen_fwd     CISGraph(128, 224, 1, with_pwc=False, train=False), bench.py --workload gen_fwd: its mask plan, then the rest of the forward
  ensemble    CISGraph(192, 384, 4, train=False), bench.py --workload ensemble: PWC-Net at batch 4, the recover net at N = 12 with split-K
              6 and 7 over batch-broadcast concats, the stride-2 phase-halo launches; mask plan, then the rest of the forward
  odd         CISGraph(100, 172, 3, with_pwc=False): fwd, bwd['R'], bwd['G'] and the BN fold, on partial 16 x 8 tiles and odd widths
  r1, r2, r3  _PWCRunner(2, 384, 640, trainable=True) at search ranges 1, 2, 3: cis_warp_costvol_r and its transpose, and at r = 1 the
              compact thin = 16 conv6_0 on the 9-channel cost volume padded to 16
  dense_off   the same network without dense connections

Inputs are seeded smooth images (and flows) and the parameters carry a 0.1 jitter (OP.make_params), so that BN statistics and biases are
not trivial.  For the two benchmarked graphs, forward_masks(use_graph=True) -- the timed path, one CUDA graph -- is then captured, every
buffer the plans write (the mask, activations, scratch; not the inputs or parameters) is filled with NaN, and then with +-2^100, as in
tests/test_glue_launches_gpu.py's poisoned replay, and the graph is replayed on the same inputs: its mask must be bit-identical to the one
the per-launch replay produced (no launch of the mask plan uses atomics).

One summary line per graph and launch kind (count, worst bound ratio, descriptor-side persistent-kernel candidates) and the controls are
printed with pytest -s.  Controls: every control made must be rejected (ratio > 1) except costvol_bwd.gate_one, whose effect vanishes
where the pyramid's correlations are almost all positive (tests/test_glue_launches_gpu.py checks it on independent random features, for
cis_warp_costvol_bwd at R = 4 and cis_warp_costvol_bwd_r at r = 1, 2, 3).

Measured on an H100 80GB HBM3 (700 W power limit): every launch within its bound, no bug found.  Conv launches checked / worst ratio:
gen_fwd 49 / 0.954, ensemble 158 / 0.988, odd 185 / 0.983 (weight gradients <= 0.029, bias and BN gradients 0.012), r1, r2, r3 and
dense_off 357 / 0.989 each.  Other launches: 0.996 at most (the bf16 resizes and their transposes, at the rounding term 2^-8 |ref|);
cis_warp_costvol_r 0.991 / 0.990 / 0.991 and cis_warp_costvol_bwd_r 0.995 / 0.994 / 0.993 at r = 1 / 2 / 3; cis_warp_costvol 0.992
(ensemble) and 0.991 (dense_off), its transpose 0.993 (dense_off).  New controls: tile.partial 7.4 - 8.0,
thin16.cin9 (conv6_0 at r = 1) 2047, thin8.cin5 (the generator's conv1) 2419 - 2995, warp_costvol_r1.dx_outer 4.1e4; gate_one
0.993 - 0.995.  Both captured mask graphs, replayed over poisoned buffers, bit-identical to the per-launch replay.  The file runs
in 20 - 32 s."""
import functools
import time

import pytest
import torch

import conv_launch_ref as R
import glue_launch_ref as G
import pwc_options_ref as REF
from oracle import params as OP
from test_glue_launches_gpu import _poison
from test_graph_variants_launches_cpu import CONV, KEYS, PWC_OPTIONS, build

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

UNREJECTED = {'costvol_bwd.gate_one'}


def _images(B, H, W, seed):
    gen = torch.Generator().manual_seed(seed)
    img1 = R.smooth(B, H, W, 3, 0.25, gen).clamp(-0.5, 0.5)
    return img1, torch.roll(img1, shifts=(2, 3), dims=(1, 2)) + 0.01 * torch.randn(B, H, W, 3, generator=gen), gen


def _inputs(key, g):
    """Parameters and inputs of graph `key`, packed."""
    if key in ('gen_fwd', 'odd'):
        g.load_params(OP.make_params(seed=4, jitter=0.1, nets=('MaskNet', 'FlownetS')))
        gen = torch.Generator().manual_seed(5)
        g.image.copy_(torch.rand(g.B, g.H, g.W, 3, generator=gen) - 0.5)
        g.flow.copy_(R.smooth(g.B, g.H, g.W, 2, 0.3, gen))
        g._ensure_packed()
    elif key == 'ensemble':
        g.load_params(OP.make_params(seed=1, jitter=0.1))
        img1, img2, _ = _images(g.B, 384, 640, 7)
        g.img1.copy_(img1)
        g.img2.copy_(img2)
        g._ensure_packed()
    else:
        g.reload(REF.make_params(1, jitter=0.1, options=PWC_OPTIONS[key]))
        img1, img2, gen = _images(g.B, g.H, g.W, 13)
        g.img1.copy_(img1)
        g.img2.copy_(img2)
        g.dflow_out.copy_(R.smooth(g.B, g.H, g.W, 2, 1.0, gen))


def _report(key, w, glue, rec, plans):
    cand = R.count_persist(rec, plans)
    for lab, v in w.summary().items():
        print('%-10s %-40s count %4d  worst bound ratio %.3g  persistent-kernel candidates %d'
              % (key, lab, v['count'], v['worst'], cand[lab][1] if lab in cand else 0))
    for lab, v in glue.summary().items():
        print('%-10s %-40s count %4d  worst bound ratio %.3g' % (key, lab, v['count'], v['worst']))
    print('%-10s negative controls (ratio > 1 = rejected): %s' % (key, dict(w.controls, **glue.controls)))


@functools.lru_cache(maxsize=None)
def walk(key):
    """Replay of graph `key` with every launch checked -> dict of plain results (the graph and its buffers are released)."""
    t0 = time.time()
    g, rec, plans = build(key, 'cuda')
    _inputs(key, g)
    glue = G.Glue(controls=True)
    w = R.Walker(rec, controls=True, glue=glue)
    out = dict(failures=[], mask=None, graph_mask=None, bn_fold=0.0)
    for name, plan in plans:
        n, m = len(w.failures), len(glue.failures)
        w.run(plan)
        out['failures'] += ['%s: %s' % (name, f) for f in w.failures[n:] + glue.failures[m:]]
        if name == 'masks':
            out['mask'] = g.mask.clone()
    if key in ('gen_fwd', 'ensemble', 'odd'):
        out['bn_fold'] = R.check_bn_fold(g.gen.all_layers())
    if out['mask'] is not None:
        # The first call captures the CUDA graph (after running the plan eagerly once); every buffer the plans write is then poisoned
        # and the second call only replays the graph, so the mask it leaves is the captured graph's own work.
        g.forward_masks(use_graph=True)
        out['graph_mask'] = {}
        for sentinel in (float('nan'), 2.0 ** 100):
            _poison(g, [], sentinel)
            torch.cuda.synchronize()
            poisoned = not torch.equal(g.mask, out['mask'])
            assert set(g.graphs) == {'masks'}
            g.forward_masks(use_graph=True)
            torch.cuda.synchronize()
            out['graph_mask'][sentinel] = (poisoned, g.mask.clone())
    _report(key, w, glue, rec, [p for _, p in plans])
    out.update(controls=dict(w.controls, **glue.controls), conv=w.checked, glue=sum(glue.counts.values()))
    print('%-10s %d conv and %d other launches checked in %.1f s' % (key, out['conv'], out['glue'], time.time() - t0))
    del g, rec, plans, w, glue
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return out


@pytest.mark.parametrize('key', KEYS)
def test_every_launch_within_its_bound(key):
    r = walk(key)
    assert not r['failures'], '%s:\n%s' % (key, '\n'.join(r['failures'][:20]))
    assert r['conv'] == CONV[key]
    assert r['bn_fold'] <= 1.0, r['bn_fold']


@pytest.mark.parametrize('key', KEYS)
def test_negative_controls_are_rejected(key):
    c = walk(key)['controls']
    want = {'tile', 'tile.partial', 'fwd.halo'}
    want |= {'thin8.cin5'} if key in ('gen_fwd', 'ensemble', 'odd') else set()          # the generator's conv1
    want |= {'thin16.cin9', 'warp_costvol_r1.dx_outer'} if key == 'r1' else set()
    want |= {'tile.cis_warp_costvol_r'} if key in ('r1', 'r2', 'r3') else set()
    assert want <= set(c), (key, sorted(want - set(c)))
    bad = {k: v for k, v in c.items() if k not in UNREJECTED and not v > 1.0}
    assert not bad, (key, bad)


@pytest.mark.parametrize('key', ['gen_fwd', 'ensemble'])
def test_timed_mask_path_is_bit_identical_to_the_checked_replay(key):
    """A replay of the captured forward_masks(use_graph=True) graph, over buffers (mask included) filled with NaN, then with +-2^100,
    against the mask the per-launch replay of _mask_plan wrote, on the same inputs and parameters."""
    r = walk(key)
    for sentinel, (poisoned, mask) in r['graph_mask'].items():
        assert poisoned, sentinel
        assert torch.equal(mask, r['mask']), sentinel
