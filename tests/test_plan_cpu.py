"""The launch planner on CPU: the whole step graph (PWC-Net + generator + 3x recover + both backward plans) is BUILT on CPU tensors --
nothing is launched -- and every conv / wgrad descriptor is checked against the rules the C-side launchers enforce
(csrc/conv_igemm.cu: cis_conv_igemm, launch_halo, launch_fwd, cis_conv_wgrad), plus the bookkeeping the bench line relies on."""
import collections

import pytest

import plan_digest
from unsupervised_detection_b200 import engine
from unsupervised_detection_b200.step_graph import CISGraph


@pytest.fixture(scope='module')
def graph():
    return CISGraph(64, 96, 1, device='cpu', global_batch=2)


def _convs(plan):
    return [a[0]._obj for fn, a, name, fl, lane in plan.ops if name == 'cis_conv_igemm']


def _check_conv(d):
    assert 1 <= d.ntaps <= 49 and 1 <= d.nsrc <= 4 and d.K_pad > 0 and d.K_pad % 64 == 0 and d.n_tiles >= 1 and d.wpack
    assert d.BN in (16, 32, 64, 128)
    chunks = 0
    for i in range(d.nsrc):
        s = d.src[i]
        assert s.ptr and (s.pitch | s.c_off) % 8 == 0 and s.chunks >= 1
        chunks += s.chunks
    assert d.ntaps * chunks * 8 <= d.K_pad or d.halo          # generic packing: taps x channels fit the padded K
    assert d.out or d.outf
    if d.out:
        assert d.out_pitch > 0 and d.out_ch >= 1     # unaligned channel offsets are legal (scalar store path), e.g. PWC up_flow slices
    if d.halo:
        assert d.sh == 1 and d.sw == 1 and 1 <= d.MT <= 4 and d.MT * d.BN <= engine.MAX_ACC_COLS and d.dil >= 1
        hp = (8 + d.ex) * (16 * d.MT + d.ey)
        assert 2 * ((hp * 128 + 1023) // 1024 * 1024) + hp * 4 + 1024 + d.BN * 128 <= 227 * 1024      # at least one weight stage fits
        hp0, wp0 = -(-d.OH // d.dil), -(-d.OW // d.dil)
        util = hp0 * wp0 / float((-(-hp0 // (16 * d.MT))) * 16 * d.MT * (-(-wp0 // 8)) * 8)
        assert util >= (0.2 if d.dil == 1 else 0.5)               # engine.HALO_MIN_UTIL; dilated phases keep the old rule
        for t in range(d.ntaps):
            assert 0 <= d.dh[t] <= d.ey and 0 <= d.dw[t] <= d.ex                                   # taps are halo-relative
        if d.MT > 1 and d.nsub <= 1 and engine.PLAN_MODEL == 4:
            # planner rule measured in r02: a taller tile stack only on big grids of short tiles (MMA loop < a CTA's fixed costs)
            n1 = d.N * d.dil * d.dil * (-(-wp0 // 8)) * (-(-hp0 // 16)) * d.n_tiles
            assert 2.0 * d.BN * d.ntaps * (-(-chunks // 8)) < 6000.0 and n1 > 4 * engine.NUM_SMS
    if d.splits > 1:                                  # two-launch split-K (default): private slices, no ticket counters, every split owns work
        assert d.sk_scratch and not d.sk_counters and 2 <= d.splits <= 16
        units = -(-chunks // 8) if d.halo else d.K_pad // 64
        assert (d.splits - 1) * (-(-units // d.splits)) < units


def test_every_conv_descriptor_is_launchable(graph):
    n = 0
    for plan in (graph.fwd, graph.bwd['G'], graph.bwd['R']):
        for d in _convs(plan):
            _check_conv(d)
            n += 1
    assert n > 250
    for plan in (graph.bwd['G'], graph.bwd['R']):
        for fn, a, name, fl, lane in plan.ops:
            if name != 'cis_conv_wgrad':
                continue
            w = a[0]._obj
            assert w.Cout <= 128 and w.K_pad % 64 == 0 and w.splits >= 1 and w.g and w.dwp and w.tma in (0, 1, 2)
            assert lane == 1                                                                       # weight gradients run on the side lane
            # the private split slices of a layer (written once, read back once by the un-pack job) stay under engine.WGRAD_MAX_SLICE_MB
            assert w.splits == 1 or w.splits * w.Cout * w.K_pad * 4 <= engine.WGRAD_MAX_SLICE_MB * 1e6
            if w.tma:
                assert w.sh == 1 and all(w.src[i].chunks % 8 == 0 for i in range(w.nsrc - 1))


def test_plan_bookkeeping(graph):
    g = graph
    assert g.param_count() == 18918722                      # "Number of params" the reference prints (adversarial_learner.py:338)
    # the generator step back-propagates through the recover net's data path but only accumulates generator weight gradients
    wg = {m: sum(1 for op in g.bwd[m].ops if op[2] == 'cis_conv_wgrad') for m in 'GR'}
    assert wg['G'] == 17 and wg['R'] == 32
    kinds = collections.Counter(op[2] for op in g.fwd.ops if op[0] is not None)
    assert kinds['cis_warp_costvol'] == 5 and kinds['cis_cis_loss_fwd'] == 1 and kinds['cis_cis_loss_reduce'] == 1
    assert g.launches_per_step('G') > 400 and g.launches_per_step('R') > 400
    flops = sum(op[3] for op in g.fwd.ops)
    assert flops > 0


def test_experiment_switches_change_only_what_they_claim(monkeypatch):
    """Two-launch split-K (on by default) and the thin-layer switch are planner decisions: preview them without a GPU."""
    monkeypatch.setattr(engine, 'SPLITK', 0)
    base = CISGraph(64, 96, 1, device='cpu', global_batch=1)
    nbase = base.fwd.count()
    assert not [d for d in _convs(base.fwd) if d.splits > 1]
    monkeypatch.setattr(engine, 'SPLITK', 2)
    monkeypatch.setattr(engine, 'SPLITK_MAX', 16)
    monkeypatch.setattr(engine, 'SPLITK_NCTA', 8)
    monkeypatch.setattr(engine, 'SPLITK_MIN_UNITS', 16)
    g = CISGraph(64, 96, 1, device='cpu', global_batch=1)
    split = [d for d in _convs(g.fwd) if d.splits > 1]
    assert split and all(not d.sk_counters and d.sk_scratch for d in split)        # NULL counters = two-launch mode
    assert g.fwd.count() == nbase + len(split)                                     # the finish launch is counted
    for d in split:
        units = (-(-sum(d.src[i].chunks for i in range(d.nsrc)) // 8)) if d.halo else d.K_pad // 64
        per = -(-units // d.splits)
        assert (d.splits - 1) * per < units                                        # every split owns at least one unit (launcher check)
    monkeypatch.setattr(engine, 'SPLITK', 0)
    monkeypatch.setattr(engine, 'HALO_SKIP_THIN', 8)
    g2 = CISGraph(64, 96, 1, device='cpu', global_batch=1)
    changed = [(a.halo, b.halo) for a, b in zip(_convs(base.fwd), _convs(g2.fwd)) if a.halo != b.halo]
    assert changed and all(a == 1 and b == 0 for a, b in changed)                  # only halo -> gather moves
    assert all(sum(d.src[i].chunks for i in range(d.nsrc)) * 8 <= 8 and d.ntaps >= 16
               for d, e in zip(_convs(base.fwd), _convs(g2.fwd)) if d.halo != e.halo)


def test_param_job_tables_follow_the_device_side_block_mapping(graph):
    """cis_param_multi's job tables (engine.Plan.batch_param_ops) against the rules the kernel applies (csrc/misc_kernels.cu:
    param_multi_kernel): first-block prefix sums, one block per 8 output channels for the BN chain rule, one block per BN x 64 tile for the
    forward-orientation tiled pack, flat 256-element blocks otherwise, and the slice layout flag of every un-pack job."""
    import ctypes as C
    from unsupervised_detection_b200._lib import CisParamJob, JOB_PACK, JOB_PACK_TILED, JOB_UNPACK, JOB_BN_FOLD, JOB_BN_CHAIN
    g = graph
    plans = [g.pack_gen, g.pack_rec, g.bwd['G'], g.bwd['R']]
    seen = set()
    slice_writer = {}          # slice buffer -> kernel path that fills it (CisWgrad.tma), from the weight-gradient launches themselves
    for m in 'GR':
        for fn, a, name, fl, lane in g.bwd[m].ops:
            if name == 'cis_conv_wgrad':
                slice_writer[a[0]._obj.dwp] = a[0]._obj.tma
    for plan in plans:
        for fn, a, name, fl, lane in plan.ops:
            if name != 'cis_param_multi':
                continue
            tab = next(t for t in plan.keep if hasattr(t, 'data_ptr') and t.data_ptr() == a[0])
            njobs, total = a[1], a[2]
            raw = bytes(tab.cpu().numpy().tobytes())
            jobs = [CisParamJob.from_buffer_copy(raw[q * C.sizeof(CisParamJob):(q + 1) * C.sizeof(CisParamJob)]) for q in range(njobs)]
            assert len({j.kind for j in jobs}) == 1                                   # one kind per launch
            first = 0
            for j in jobs:
                assert j.i[7] == first
                if j.kind == JOB_BN_CHAIN:
                    blocks = -(-j.i[0] // 8)
                elif j.kind == JOB_PACK_TILED:
                    cin8, ntaps, n_tiles, BN, cout, sn = (j.i[q] for q in range(6))
                    tiles = n_tiles * (-(-cin8 // 64)) * ntaps
                    blocks = tiles if sn == 1 else -(-(tiles * BN * 64) // 256)
                    assert BN <= 128
                elif j.kind == JOB_UNPACK:
                    K_pad, cout, nsplit, nblocks, nch, layout = (j.i[q] for q in range(6))
                    blocks = -(-(cout * K_pad + nch) // 256)
                    assert layout in (0, 1) and K_pad % 4 == 0 and nsplit >= 1 and 1 <= nblocks <= 592
                    assert layout == (0 if slice_writer[j.p[0]] == 2 else 1)          # reader and writer agree on the slice layout
                elif j.kind == JOB_PACK:
                    blocks = -(-(j.i[1] * j.i[0]) // 256)
                else:
                    assert j.kind == JOB_BN_FOLD
                    blocks = -(-max(j.n, j.i[0]) // 256)
                first += blocks
                seen.add(j.kind)
            assert first == total
    assert seen == {JOB_PACK, JOB_PACK_TILED, JOB_UNPACK, JOB_BN_FOLD, JOB_BN_CHAIN}


def test_plan_digest_is_stable_across_builds():
    """Two builds of the same graph and of the same layer runner give the same canonical plans (tests/plan_digest.py): the check
    that a change to the plan builders leaves every launch, pointer target and packed table as it was relies on it."""
    from unsupervised_detection_b200.models import functional as F
    spec = ('gen', 1, 16, 2, 1, engine.ACT_ELU, None, None, 'Net/l')       # stride-2 1x1: tapless output parities
    digests = []
    for _ in range(2):
        with plan_digest.filled_uninitialized():
            g = CISGraph(64, 96, 1, device='cpu', pwc_hw=(128, 192))
            r = F._LayerRunner(2, 37, 53, 20, spec, 'cpu')
            r.ensure_backward()
        digests.append((plan_digest.digest(plan_digest.graph_plans(g)), plan_digest.digest(plan_digest.runner_plans(r))))
    assert digests[0] == digests[1]
    assert any(line.startswith('cis_conv_wgrad') for line in digests[0][0])
