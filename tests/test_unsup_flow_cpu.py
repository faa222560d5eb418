"""Unsupervised PWC-Net fine-tuning without a GPU: the fp64 restatement of the census + smoothness loss (tests/unsup_flow_loss_ref.py)
against hand-computed cases, the folded census gradient the backward kernel gathers, the launch lists of FlowTrainGraph(loss=
'unsupervised'), and the usage of train_flow.py --flow_loss=unsupervised."""
import collections
import os
import sys

import pytest
import torch

import unsup_flow_loss_ref as UR
from chairs_tree import make_chairs_tree
from flow_trees import make_davis_tree, make_tree
from unsupervised_detection_b200.flow_train_graph import FlowTrainGraph

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NONDENSE = {'use_dense_cx': False, 'use_res_cx': False, 'search_range': 2}
D = torch.float64


def _frames(B, H, W, seed, pad=0):
    gen = torch.Generator().manual_seed(seed)
    return torch.rand(B, H + 2 * pad, W + 2 * pad, 3, generator=gen, dtype=D) - 0.5


# ------------------------------------------------------------------------------------------------ the loss restated
def test_identical_frames_and_zero_flow():
    a = _frames(2, 12, 15, 0)
    flow = torch.zeros(4, 12, 15, 2, dtype=D)
    s, t = UR.direction_sums(flow, a, a)
    # c = 0 up to the last bits of the warp's clamped last row and column (alpha = 1: tl + 1 * (tr - tl))
    assert torch.equal(t['M'], torch.ones_like(t['M'])) and float(t['c'].abs().max()) <= 1e-25
    assert torch.equal(s[:, 1], torch.zeros(4, dtype=D))
    # c = 0 everywhere: the census term sits at its floor psi(0) = 0.01^0.4 per pixel
    assert torch.allclose(s[:, 0], torch.full((4,), 12 * 15 * 0.01 ** 0.4, dtype=D), rtol=1e-12, atol=0)


@pytest.mark.parametrize('dy,dx', [(2, -3), (0, 1), (-1, 0)])
def test_integer_translation_with_exact_flows(dy, dx):
    """frame 2 = frame 1 moved by (dy, dx): the forward flow is -(dy, dx), the backward one +(dy, dx) (PWC-Net's order and sign)."""
    B, H, W, m = 2, 14, 17, 4
    big = _frames(B, H, W, 1, pad=m)
    img1 = big[:, m:m + H, m:m + W]
    img2 = big[:, m - dy:m - dy + H, m - dx:m - dx + W]
    flow = torch.cat([torch.tensor([-dy, -dx], dtype=D).expand(B, H, W, 2), torch.tensor([dy, dx], dtype=D).expand(B, H, W, 2)]).contiguous()
    M, V, _, _ = UR.mask(flow)
    _, t = UR.direction_sums(flow, img1, img2)
    y = torch.arange(H).view(H, 1).expand(H, W)
    x = torch.arange(W).view(1, W).expand(H, W)
    for n, (sy, sx) in enumerate([(dy, dx)] * B + [(-dy, -dx)] * B):
        inside = (y + sy >= 0) & (y + sy <= H - 1) & (x + sx >= 0) & (x + sx <= W - 1)      # q = p + (sy, sx)
        assert torch.equal(V[n].bool(), inside) and torch.equal(M[n].bool(), inside)          # V = 0 exactly on the band that leaves
        # c = 0 wherever the whole window (inside the frame) samples inside the frame
        ok = torch.zeros(H, W, dtype=torch.bool)
        for yy in range(H):
            for xx in range(W):
                ok[yy, xx] = bool(inside[max(0, yy - 3):yy + 4, max(0, xx - 3):xx + 4].all())
        assert ok.any() and float(t['c'][n][ok].abs().max()) <= 1e-25
        assert float(t['c'][n][~inside].max()) > 0                                             # off the frame: clamped, not matched


def test_occlusion_threshold_by_hand():
    f = torch.tensor([1.0, 0.0], dtype=D)
    lhs, rhs = UR.occlusion_terms(f, torch.tensor([-1.0, 0.0], dtype=D))
    assert float(lhs) == 0.0 and float(rhs) == pytest.approx(0.52) and not lhs > rhs          # consistent: visible
    lhs, rhs = UR.occlusion_terms(f, torch.tensor([0.0, 0.0], dtype=D))
    assert float(lhs) == 1.0 and float(rhs) == pytest.approx(0.51) and lhs > rhs              # partner static: occluded
    # the same through mask(): forward flow (1, 0) everywhere, backward (-1, 0) or (0, 0)
    H, W = 6, 7
    fw = torch.tensor([1.0, 0.0], dtype=D).expand(1, H, W, 2)
    for bw, occluded in ((torch.tensor([-1.0, 0.0], dtype=D), False), (torch.zeros(2, dtype=D), True)):
        M, V, _, _ = UR.mask(torch.cat([fw, bw.expand(1, H, W, 2)]).contiguous())
        assert torch.equal(V[0, 1:], torch.ones(H - 1, W, dtype=D)) and torch.equal(V[0, 0], torch.zeros(W, dtype=D))   # q_y = y - 1
        assert torch.equal(M[0], torch.zeros(H, W, dtype=D) if occluded else V[0])


def test_smoothness_affine_is_zero_and_quadratic_by_hand():
    H, W = 9, 11
    y = torch.arange(H, dtype=D).view(1, H, 1).expand(1, H, W)
    x = torch.arange(W, dtype=D).view(1, 1, W).expand(1, H, W)
    S = (0.01 * y).unsqueeze(-1).expand(1, H, W, 3).contiguous() - 0.4     # a vertical ramp: |S(y+1) - S(y-1)| = 0.02 per channel
    affine = torch.stack([0.5 + 0.25 * y - 1.5 * x, -2.0 + 0.75 * x + 0.125 * y], -1)
    assert float(UR.smoothness(affine, S)) == 0.0
    quad = torch.stack([y * y, torch.zeros_like(y)], -1)                    # second difference 2 along y, 0 along x
    want = (H - 2) * W * 2.0 * torch.exp(torch.tensor(-10.0 * 0.02 / 2, dtype=D))
    assert abs(float(UR.smoothness(quad, S)) - float(want)) <= 1e-12 * float(want)
    # edge weights: the same flow on a vertical ramp 10x steeper weighs each term exp(-1)
    assert abs(float(UR.smoothness(quad, 10 * (S + 0.4))) - float((H - 2) * W * 2.0 * torch.exp(torch.tensor(-1.0, dtype=D)))) <= 1e-12


def test_psi_and_its_gradient_are_finite_at_zero():
    c = torch.zeros(3, dtype=D, requires_grad=True)
    p = UR.psi(c)
    (g,) = torch.autograd.grad(p.sum(), c)
    assert torch.allclose(p, torch.full((3,), 0.01 ** 0.4, dtype=D)) and torch.allclose(g, torch.full((3,), 0.4 * 0.01 ** -0.6, dtype=D))


def test_loss_is_divided_by_global_batch_and_pixels():
    B, H, W = 2, 10, 12
    a, b = _frames(B, H, W, 3), _frames(B, H, W, 4)
    gen = torch.Generator().manual_seed(5)
    flow = torch.randn(2 * B, H, W, 2, generator=gen, dtype=D)
    s, _ = UR.direction_sums(flow, a, b)
    for gb, lam in ((B, 3.0), (8, 0.5)):
        want = (s[:, 0].sum() + lam * s[:, 1].sum()) / (gb * H * W)
        assert abs(float(UR.loss(flow, a, b, global_batch=gb, smooth_weight=lam)) - float(want)) <= 1e-15 * abs(float(want))


def test_census_gradient_is_the_folded_window_gather():
    """The backward kernel's census gather: dT~(r) = -sum_d (k(r+d) + k(r)) h(r, r+d), against autograd of sum M psi(c) in T~."""
    gen = torch.Generator().manual_seed(6)
    N, H, W = 2, 9, 13
    gs = torch.rand(N, H, W, generator=gen, dtype=D) * 40
    tw = (gs + torch.randn(N, H, W, generator=gen, dtype=D) * 3).requires_grad_(True)
    m = (torch.rand(N, H, W, generator=gen, dtype=D) > 0.3).to(D)
    c = UR.census(gs, tw)
    (ref,) = torch.autograd.grad((m * UR.psi(c)).sum(), tw)
    k = (m * 0.4 * (c + 0.01) ** -0.6).detach()
    t = tw.detach()
    got = torch.zeros_like(t)
    for dy in range(-3, 4):
        for dx in range(-3, 4):
            if dy == 0 and dx == 0:
                continue
            s2, ins = UR._shift(gs, dy, dx)
            t2, _ = UR._shift(t, dy, dx)
            k2, _ = UR._shift(k, dy, dx)
            u = t2 - t
            iu = 1 / torch.sqrt(0.81 + u * u)
            d = (s2 - gs) / torch.sqrt(0.81 + (s2 - gs) ** 2) - u * iu
            h = -0.2 * d / (0.1 + d * d) ** 2 * 0.81 * iu ** 3
            got -= ins * (k2 + k) * h
    assert torch.allclose(got, ref, rtol=1e-10, atol=1e-12)


# ------------------------------------------------------------------------------------------------ the training graph's launch lists
def _counts(plan):
    return collections.Counter(op[2] for op in plan.ops)


@pytest.mark.parametrize('options', [None, NONDENSE])
def test_unsupervised_graph_launches(options):
    B, H, W, GB = 2, 128, 192, 4
    g = FlowTrainGraph(H, W, B, options=options, device='cpu', global_batch=GB, loss='unsupervised', smooth_weight=2.0)
    total = collections.Counter()
    for p in (g.fwd, g.bwd, g.adam, g.pack):
        total += _counts(p)
    assert total['cis_flow_multiscale_loss'] == 0 and total['cis_flow_multiscale_loss_bwd'] == 0
    assert total['cis_unsup_flow_loss'] == 1 and total['cis_unsup_flow_loss_bwd'] == 1 and total['cis_adam_l2'] == 1
    # four packs into the halves of the two 2B image Acts: (img1, img2) then (img2, img1)
    packs = [op[1] for op in g.fwd.ops if op[2] == 'cis_pack_f32_to_bf16']
    i1, i2 = g.img_acts
    half = B * H * W * 8 * 2
    assert i1.N == i2.N == 2 * B
    assert [(a[0], a[1], a[4]) for a in packs] == [(g.img1.data_ptr(), B * H * W, i1.ptr), (g.img2.data_ptr(), B * H * W, i1.ptr + half),
                                                 (g.img2.data_ptr(), B * H * W, i2.ptr), (g.img1.data_ptr(), B * H * W, i2.ptr + half)]
    # the loss forward is the last launch, on the final flow of the 2B batch and the fp32 frames
    last = g.fwd.ops[-1]
    assert last[2] == 'cis_unsup_flow_loss' and last[1][:6] == (g.flow.data_ptr(), g.img1.data_ptr(), g.img2.data_ptr(), B, H, W)
    assert tuple(g.flow.shape) == (2 * B, H, W, 2) and tuple(g.sums.shape) == (2 * B, 2)
    # seed: zero the level gradients, the loss backward, the final x4 resize's transpose into the level-2 flow gradient
    names = [op[2] for op in g.bwd.ops]
    nz = len(g.pwc.level_grad)
    assert names[:nz + 2] == ['cis_zero'] * nz + ['cis_unsup_flow_loss_bwd', 'cis_resize_f32_bwd_to_bf16_scaled']
    bwd = g.bwd.ops[nz][1]
    assert bwd[8] == pytest.approx(1.0 / (GB * H * W), rel=1e-7) and bwd[9] == pytest.approx(2.0 / (GB * H * W), rel=1e-7)
    assert bwd[10] == g.dflow.data_ptr()
    fg = g.pwc.flows_bf[2].get_grad()
    assert g.bwd.ops[nz + 1][1] == (g.dflow.data_ptr(), 2 * B, H, W, 2, H // 4, W // 4, fg.ptr, fg.pitch, 4.0)
    # no conv1a data gradient
    for a in g.img_acts:
        assert a.grad is None and not a.grad_written and not a.dep
    # cis_adam_l2 as in the supervised graph
    sup = FlowTrainGraph(H, W, B, options=options, device='cpu', global_batch=GB)
    assert [op[2] for op in g.adam.ops] == ['cis_adam_l2']
    assert g.adam.ops[0][1][4:] == sup.adam.ops[0][1][4:5] + (g._seg.data_ptr(),) + sup.adam.ops[0][1][6:8] + (g.lr.data_ptr(),) + \
        sup.adam.ops[0][1][9:12] + (g.step_state.data_ptr(),)
    assert g.kernel_seg == sup.kernel_seg
    # the same network and reverse tape as the supervised step, less the loss: the launch lists differ only there
    diff = _counts(g.fwd) + _counts(g.bwd)
    diff.subtract(_counts(sup.fwd) + _counts(sup.bwd))
    assert {k: v for k, v in diff.items() if v} == {'cis_pack_f32_to_bf16': 2, 'cis_flow_multiscale_loss': -1, 'cis_unsup_flow_loss': 1,
                                                     'cis_flow_multiscale_loss_bwd': -1, 'cis_unsup_flow_loss_bwd': 1,
                                                     'cis_resize_f32_bwd_to_bf16_scaled': 1}


def test_unsupervised_graph_arguments():
    with pytest.raises(ValueError):
        FlowTrainGraph(128, 128, 1, device='cpu', loss='unsupervised', smooth_weight=-1.0)
    g = FlowTrainGraph(128, 128, 1, device='cpu', in_hw=(384, 640), loss='unsupervised')
    assert _counts(g.fwd)['cis_resize_bilinear_f32'] == 3                # the two frames to 128x128, the final x4
    res = [op[1] for op in g.fwd.ops if op[2] == 'cis_resize_bilinear_f32'][:2]
    loss = [op[1] for op in g.fwd.ops if op[2] == 'cis_unsup_flow_loss'][0]
    assert loss[1:3] == (res[0][5], res[1][5])                            # the loss reads the resized frames
    sup = FlowTrainGraph(128, 128, 1, device='cpu')
    with pytest.raises(ValueError):
        sup.feed(torch.zeros(1, 128, 128, 3), torch.zeros(1, 128, 128, 3))   # the supervised loss needs the ground truth


# ------------------------------------------------------------------------------------------------ train_flow.py
def test_train_flow_unsupervised_usage(monkeypatch, tmp_path):
    sys.path.insert(0, ROOT)
    import train_flow as TF
    from unsupervised_detection_b200.common_flags import FLAGS, FLAG_NAMES
    assert 'smooth_weight' in TF.TRAIN_FLOW_FLAGS and not set(TF.TRAIN_FLOW_FLAGS) & set(FLAG_NAMES)
    roots = {ds: make_tree(ds, tmp_path / ds.lower()) for ds in ('DAVIS2016', 'FBMS', 'SEGTRACK')}
    roots['FLYINGCHAIRS'] = make_chairs_tree(tmp_path / 'chairs', n=2, labels=[1, 2])
    noval = make_davis_tree(tmp_path / 'noval', seqs=(('train', ('bear',)),))
    seen = []
    monkeypatch.setattr(TF, 'run', lambda cfg: seen.append((cfg.dataset, cfg.flow_loss, cfg.smooth_weight, cfg.validate)))
    ck = '--checkpoint_dir=%s' % (tmp_path / 'ck')

    def main(*args):
        FLAGS.unparse_flags()
        TF.main(['train_flow.py', ck, '--flow_loss=unsupervised'] + list(args))
    try:
        for ds, root in sorted(roots.items()):
            main('--dataset=' + ds, '--root_dir=' + root, '--validate')
        main('--dataset=DAVIS2016', '--root_dir=' + roots['DAVIS2016'], '--smooth_weight=0')
        main('--dataset=DAVIS2016', '--root_dir=' + noval)                                     # no val pairs, no --validate: fine
        assert seen == [(ds, 'unsupervised', 3.0, True) for ds in sorted(roots)] + [('DAVIS2016', 'unsupervised', 0.0, False),
                                                                                   ('DAVIS2016', 'unsupervised', 3.0, False)]
        fdir = tmp_path / 'flo'
        fdir.mkdir()
        bad = [['--dataset=DAVIS2016', '--root_dir=' + roots['DAVIS2016'], '--flow_dir=%s' % fdir],   # --flow_dir replaces PWC-Net
               ['--dataset=DAVIS2016', '--root_dir=' + roots['DAVIS2016'], '--smooth_weight=-0.5'],
               ['--dataset=DAVIS2016', '--root_dir=' + noval, '--validate'],                          # no val pairs
               ['--dataset=SYNTHETIC']]
        for b in bad:
            with pytest.raises(SystemExit):
                main(*b)
    finally:
        FLAGS.unparse_flags()
    assert len(seen) == 6
