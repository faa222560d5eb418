"""Augmentation of supervised PWC-Net training pairs on the GPU: cis_flow_aug_params and cis_flow_augment against the fp64 restatement
(tests/flow_aug_ref.py), the consistency of the augmented flow with the augmented frames, FlowTrainGraph(augment=True) under CUDA graphs,
unaugmented validation, and train_flow.py --flow_aug end to end."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import flow_aug_ref as AR  # noqa: E402
from chairs_tree import make_chairs_tree  # noqa: E402
from unsupervised_detection_b200 import _lib  # noqa: E402
from unsupervised_detection_b200.flow_train_graph import AUG_SEED, FlowTrainGraph, flow_aug_ranges  # noqa: E402
from unsupervised_detection_b200.params_init import init_pwcnet  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
EPS = 2.0 ** -24


def _st():
    return torch.cuda.current_stream().cuda_stream


def _smooth(B, H, W, C, amp, seed):
    gen = torch.Generator().manual_seed(seed)
    lo = torch.randn(B, C, max(2, H // 24), max(2, W // 24), generator=gen)
    return (torch.nn.functional.interpolate(lo, size=(H, W), mode='bicubic', align_corners=False) * amp).permute(0, 2, 3, 1).contiguous()


def _params(ranges, B, H, W, offset, t, seed=AUG_SEED):
    step = torch.tensor([t], dtype=torch.int64, device='cuda')
    out = torch.full((B, _lib.FLOW_AUG_ROW), float('nan'), device='cuda')
    r = flow_aug_ranges(**ranges)
    _lib.call('cis_flow_aug_params', C.byref(r), B, H, W, offset, step.data_ptr(), seed, out.data_ptr(), _st())
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _augment(img1, img2, gt, table):
    B, H, W = gt.shape[:3]
    outs = [torch.full_like(t, float('nan')) for t in (img1, img2, gt)]
    p = torch.from_numpy(table).cuda()
    _lib.call('cis_flow_augment', img1.data_ptr(), img2.data_ptr(), gt.data_ptr(), p.data_ptr(), B, H, W, *(o.data_ptr() for o in outs), _st())
    torch.cuda.synchronize()
    return [o.cpu().numpy().astype(np.float64) for o in outs]


# ------------------------------------------------------------------------------------------------ 1. the parameter draws
@pytest.mark.parametrize('t', [0, 12345])
def test_params_match_the_reference(t):
    B, H, W = 8, 384, 640
    got = _params({}, B, H, W, 0, t)
    ref = AR.params({}, B, H, W, 0, t, AUG_SEED)
    assert np.array_equal(got[:, 26], ref[:, 26])                                  # the same accept / reject choices
    assert np.array_equal(got[:, 25].view(np.uint32).astype(np.float64), ref[:, 25])  # the noise key, bit for bit
    assert np.array_equal(got[:, 27:], np.zeros((B, 5), np.float32))
    cols = list(range(25))
    ref32 = ref[:, cols].astype(np.float32).astype(np.float64)
    ulp = np.spacing(np.abs(ref32).astype(np.float32)).astype(np.float64)
    err = np.abs(got[:, cols] - ref32)
    print('MEASURED params vs fp64: attempts %s, max |diff| / ulp %.1f' % (got[:, 26].astype(int).tolist(), float((err / ulp).max())))
    assert (err <= ulp).all()                                                      # fp32 rounding of the same double
    # rows depend only on the global sample index
    part = _params({}, 3, H, W, 5, t)
    assert np.array_equal(part.view(np.uint32), got[5:8].view(np.uint32))


# ------------------------------------------------------------------------------------------------ 2. the per-pixel pass
def _frames(B, H, W, seed):
    return (_smooth(B, H, W, 3, 0.3, seed).clamp(-0.5, 0.5), _smooth(B, H, W, 3, 0.3, seed + 1).clamp(-0.5, 0.5),
            _smooth(B, H, W, 2, 6.0, seed + 2))


def _lip(a):
    """max |difference| between neighbouring pixels of a [H, W, C] field: its Lipschitz bound per pixel of the bilinear sample."""
    return max(float(np.abs(np.diff(a, axis=0)).max()), float(np.abs(np.diff(a, axis=1)).max()))


def _pos_err(m, H, W):
    """bound on the fp32 error of r0 x + r1 y + r2 (and the second row) over the grid"""
    return 4 * EPS * max(abs(m[0]) * W + abs(m[1]) * H + abs(m[2]), abs(m[3]) * W + abs(m[4]) * H + abs(m[5]))


def _check_pass(img1, img2, gt, table):
    B, H, W = gt.shape[:3]
    got = _augment(img1.cuda(), img2.cuda(), gt.cuda(), table)
    P = AR.table_rows(table)
    a1, a2, g = (t.numpy().astype(np.float64) for t in (img1, img2, gt))
    ref = AR.augment(a1, a2, g, P)
    worst = [0.0, 0.0, 0.0]
    for b in range(B):
        r = P[b]
        y, x = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing='ij')
        for f, (src, m) in enumerate(((a1[b], r[0:6]), (a2[b], r[6:12]))):
            # the sample moves by at most 2 * position error * Lipschitz bound; the affine part of the chain scales it by m_c (1 + kappa),
            # gamma maps the interval around the pre-gamma value; fp32 arithmetic adds a few ulps of 1
            qx, qy = AR.apply(m, x, y)
            s = AR.bilinear(src, qx, qy)
            pre = 0.5 + r[21] * ((s + 0.5) * r[18:21] - 0.5) + r[22]
            e = np.abs(r[21] * r[18:21]) * 2 * _pos_err(m, H, W) * _lip(src) + 1e-6
            g_ = lambda v: np.clip(v, 0, 1) ** r[23]  # noqa: E731
            tol = g_(pre + e) - g_(pre - e) + 8e-6
            d = np.abs(got[f][b] - ref[f][b])
            assert (d <= tol).all(), (b, f, float(d.max()))
            worst[f] = max(worst[f], float((d / tol).max()))
        # flow: q moves by dq; gt at q by 2 dq Lip(gt); T2^-1 scales the sum by its row norm and adds its own rounding; then - p
        dq = _pos_err(r[0:6], H, W)
        s_max = float(max(W, H) + np.abs(g[b]).max())
        inv = r[12:18]
        row = max(abs(inv[0]) + abs(inv[1]), abs(inv[3]) + abs(inv[4]))
        tol = row * (dq + 2 * dq * _lip(g[b]) + 4 * EPS * s_max) + 4 * EPS * (row * s_max + max(abs(inv[2]), abs(inv[5]))) + 2 * EPS * max(W, H)
        d = np.abs(got[2][b] - ref[2][b])
        assert (d <= tol).all(), (b, float(d.max()), tol)
        worst[2] = max(worst[2], float(d.max() / tol))
    return worst


@pytest.mark.parametrize('B,H,W,noise', [(4, 384, 640, True), (4, 384, 640, False), (3, 66, 130, True)])
def test_augment_matches_fp64(B, H, W, noise):
    ranges = {} if noise else {'noise': (0.0, 0.0)}
    table = _params(ranges, B, H, W, 0, 3)
    assert (table[:, 24] > 0).all() == noise
    worst = _check_pass(*_frames(B, H, W, 10), table)
    print('MEASURED cis_flow_augment %dx%dx%d noise=%s: worst |diff| / tolerance img1 %.3f img2 %.3f flow %.3f' % ((B, H, W, noise) + tuple(worst)))


def test_flow_is_consistent_with_the_frames():
    """frame 2 = frame 1 warped by a known smooth flow; after augmentation without photometric change, frame 2 warped by the augmented
    flow gives frame 1 again on interior pixels.  A sign or channel-order mistake shows as an O(1) error."""
    B, H, W = 2, 192, 320
    y, x = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing='ij')

    def f(px, py):                                   # frame 2's content, smooth (wavelengths of 40+ pixels)
        return np.stack([0.2 * np.sin(px / 9.0 + py / 13.0), 0.2 * np.cos(px / 11.0 - py / 7.0), 0.15 * np.sin((px + py) / 15.0)], -1)
    u = 3.0 * np.sin(y / 30.0) + 1.5
    v = -2.0 * np.cos(x / 40.0)
    img2 = f(x, y)
    img1 = f(x + u, y + v)                           # img1(p) = img2(p + (u, v))
    gt = np.stack([-v, -u], -1)
    to = lambda a: torch.from_numpy(np.repeat(a[None], B, 0)).float().contiguous()  # noqa: E731
    table = _params(AR.NO_PHOTO, B, H, W, 0, 1)
    o1, o2, og = _augment(to(img1).cuda(), to(img2).cuda(), to(gt).cuda(), table)
    errs, ctrl = [], []
    for b in range(B):
        u2, v2 = -og[b][..., 1], -og[b][..., 0]
        px, py = x + u2, y + v2
        inside = (px >= 2) & (px <= W - 3) & (py >= 2) & (py <= H - 3) & (x >= 2) & (x <= W - 3) & (y >= 2) & (y <= H - 3)
        errs.append(np.abs(AR.bilinear(o2[b], px, py) - o1[b])[inside])
        ctrl.append(np.abs(AR.bilinear(o2[b], x + v2, y + u2) - o1[b])[inside])     # channels swapped
    e, c = np.concatenate(errs), np.concatenate(ctrl)
    print('MEASURED flow consistency: mean |diff| %.2e, max %.2e; channel-swapped control mean %.2e (zooms %s)'
          % (e.mean(), e.max(), c.mean(), (1 / np.hypot(table[:, 0], table[:, 3])).round(2).tolist()))
    assert e.mean() < 3e-3 and e.max() < 3e-2 and c.mean() > 10 * e.mean()


# ------------------------------------------------------------------------------------------------ 3. the training graph
def _batches(n, B, H, W, seed):
    return [tuple(t.clone() for t in _frames(B, H, W, seed + 3 * k)) for k in range(n)]


def test_augmented_step_is_deterministic_graph_replay_identical_and_redraws():
    B, H, W = 2, 128, 128
    batches = _batches(4, B, H, W, 20)
    runs = []
    for use_graph in (False, False, True):
        g = FlowTrainGraph(H, W, B, augment=True, sample_offset=3)
        g.load_params(init_pwcnet(g.store.entries))
        tables, losses = [], []
        for b in batches:
            g.feed(*(t.cuda() for t in b))
            g.train_step(use_graph=use_graph)
            tables.append(g.aug_params.cpu().clone())
            losses.append(g.losses())
        torch.cuda.synchronize()
        runs.append(({k: v.cpu() for k, v in g.export_params().items()}, losses, tables))
    for other in runs[1:]:
        assert other[1] == runs[0][1]
        assert all(torch.equal(a, b) for a, b in zip(other[2], runs[0][2]))
        diff = [k for k in runs[0][0] if not torch.equal(runs[0][0][k], other[0][k])]
        assert not diff, diff[:5]
    tabs = runs[0][2]
    assert all(not torch.equal(tabs[k], tabs[k + 1]) for k in range(len(tabs) - 1))   # each step draws new parameters
    # the step's table is cis_flow_aug_params at Adam step k and global samples 3, 4
    for k in (0, 2):
        assert torch.equal(tabs[k], torch.from_numpy(_params({}, B, H, W, 3, k)))


def test_validation_is_not_augmented():
    """epe() after forward() is the same, bit for bit, with augmentation on or off, also after augmented train steps."""
    B, H, W = 2, 128, 192
    graphs = [FlowTrainGraph(H, W, B, augment=a) for a in (False, True)]
    p = init_pwcnet(graphs[0].store.entries)
    for b in _batches(2, B, H, W, 40):
        graphs[1].feed(*(t.cuda() for t in b))
        graphs[1].train_step(use_graph=True)
    val = [t.cuda() for t in _batches(1, B, H, W, 50)[0]]
    out = []
    for g in graphs:
        g.load_params(p)
        g.feed(*val)
        g.forward()
        out.append((g.epe().cpu().clone(), g.flow.cpu().clone()))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])
    assert torch.equal(graphs[1].batch[2].cpu(), val[2].cpu())


def test_train_flow_script_with_flow_aug(tmp_path, capsys):
    root = make_chairs_tree(tmp_path / 'chairs', n=4, labels=[1, 1, 2, 2])
    ck = tmp_path / 'ck'
    cmd = [sys.executable, os.path.join(ROOT, 'train_flow.py'), '--dataset=FLYINGCHAIRS', '--root_dir=%s' % root, '--validate', '--flow_aug',
           '--img_height=128', '--img_width=128', '--batch_size=2', '--num_samples_train=2', '--max_epochs=1', '--save_freq=1',
           '--summary_freq=1', '--num_threads=2', '--checkpoint_dir=%s' % ck]
    r = subprocess.run(cmd, env=dict(os.environ, PYTHONPATH=ROOT), cwd=str(tmp_path), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    assert "'flow_aug': True" in r.stdout and 'Training completed successfully' in r.stdout, r.stdout[-2000:]
    for suf in ('.index', '.data-00000-of-00001', '.pt'):
        assert (ck / ('pwcnet-1' + suf)).is_file(), suf
    from unsupervised_detection_b200.common_flags import Config
    from unsupervised_detection_b200.models.adversarial_learner import AdversarialLearner
    L = AdversarialLearner()
    L.config = Config(dataset='SYNTHETIC', flow_ckpt=str(ck / 'pwcnet-1'), img_height=64, img_width=96, batch_size=2)
    L.build_train_graph()
    assert 'Flow net loaded from' in capsys.readouterr().out


def test_argument_errors_launch_nothing():
    B, H, W = 2, 16, 24
    img, gt = torch.zeros(B, H, W, 3, device='cuda'), torch.zeros(B, H, W, 2, device='cuda')
    outs = [torch.full_like(t, 7.0) for t in (img, img, gt)]
    table = torch.full((B, _lib.FLOW_AUG_ROW), 7.0, device='cuda')
    step = torch.zeros(1, dtype=torch.int64, device='cuda')
    lib = _lib.load()
    r = flow_aug_ranges()
    gt_odd = gt.view(-1)[1:].data_ptr()
    bad = [('cis_flow_aug_params', (C.byref(r), 0, H, W, 0, step.data_ptr(), 1, table.data_ptr())),
           ('cis_flow_aug_params', (C.byref(r), B, 1, W, 0, step.data_ptr(), 1, table.data_ptr())),
           ('cis_flow_aug_params', (C.byref(r), B, H, W, -1, step.data_ptr(), 1, table.data_ptr())),
           ('cis_flow_aug_params', (C.byref(flow_aug_ranges(scale=(0.0, 1.0))), B, H, W, 0, step.data_ptr(), 1, table.data_ptr())),
           ('cis_flow_augment', (img.data_ptr(), img.data_ptr(), gt_odd, table.data_ptr(), B, H, W) + tuple(o.data_ptr() for o in outs)),
           ('cis_flow_augment', (img.data_ptr(), img.data_ptr(), gt.data_ptr(), table.data_ptr(), 70000, H, W) + tuple(o.data_ptr() for o in outs)),
           ('cis_flow_augment', (img.data_ptr(), img.data_ptr(), gt.data_ptr(), table.data_ptr(), B, H, 1) + tuple(o.data_ptr() for o in outs)),
           ('cis_flow_augment', (img.data_ptr(), None, gt.data_ptr(), table.data_ptr(), B, H, W) + tuple(o.data_ptr() for o in outs))]
    for name, args in bad:
        assert getattr(lib, name)(*args, _st()) == 1, name
    torch.cuda.synchronize()
    assert all(bool((t == 7.0).all()) for t in outs + [table])
