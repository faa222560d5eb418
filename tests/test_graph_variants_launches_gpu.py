"""Every launch of the graphs the project ships besides the three of tests/test_conv_launches_gpu.py, checked on its own against an fp64
reference: the conv launches by tests/conv_launch_ref.py, the others by tests/glue_launch_ref.py, in one replay per graph
(launch_suites.walk_graph; tests/test_glue_launches_gpu.py asserts on the same walk of `odd`), with every negative control of both
checkers.  The graphs and why each one (tests/test_graph_variants_launches_cpu.py pins their launch census):

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
import pytest
import torch

from launch_suites import CONV, UNREJECTED, VARIANTS, assert_within_bounds, walk_graph

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]


@pytest.mark.parametrize('key', VARIANTS)
def test_every_launch_within_its_bound(key):
    r = walk_graph(key)
    assert_within_bounds(r)
    assert r['conv'] == CONV[key]
    assert r['bn_fold'] <= 1.0, r['bn_fold']


@pytest.mark.parametrize('key', VARIANTS)
def test_negative_controls_are_rejected(key):
    c = walk_graph(key)['controls']
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
    r = walk_graph(key)
    for sentinel, (poisoned, mask) in r['graph_mask'].items():
        assert poisoned, sentinel
        assert torch.equal(mask, r['mask']), sentinel
