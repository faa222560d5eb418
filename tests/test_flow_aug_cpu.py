"""Augmentation of supervised PWC-Net training pairs without a GPU: the fp64 restatement (tests/flow_aug_ref.py) against hand-checkable
cases, the acceptance rule of the geometry draws, the C struct and argument checks, the launch lists of FlowTrainGraph(augment=True),
and train_flow.py --flow_aug."""
import ctypes as C
import math
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

import flow_aug_ref as AR
from chairs_tree import make_chairs_tree
from unsupervised_detection_b200 import _lib
from unsupervised_detection_b200.flow_train_graph import AUG_RANGES, FlowTrainGraph, flow_aug_ranges

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H, W = 48, 80


def _smooth(B, h, w, c, amp, seed):
    gen = torch.Generator().manual_seed(seed)
    lo = torch.randn(B, c, 4, 6, generator=gen, dtype=torch.float64)
    return (torch.nn.functional.interpolate(lo, size=(h, w), mode='bicubic', align_corners=False) * amp).permute(0, 2, 3, 1).numpy()


def _run(geom, gt, photo=None):
    """AR.augment of a 1-sample batch with the geometry (T1, T2) and no photometric change (or the row fields in photo)."""
    t1, t2 = geom
    P = AR.row(t1, t2, **(photo or {}))[None]
    img = np.zeros(gt.shape[:3] + (3,))
    return AR.augment(img, img, gt, P)


# ------------------------------------------------------------------------------------------------ the geometry restated
def test_translation_resamples_the_flow_and_keeps_its_values():
    gt = _smooth(1, H, W, 2, 3.0, 0)
    tx, ty = 5.0, -3.0
    _, _, out = _run(AR.geometry(H, W, t=(tx, ty)), gt)
    y, x = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing='ij')
    want = AR.bilinear(gt[0], x + tx, y + ty)
    assert np.abs(out[0] - want).max() <= 1e-12


@pytest.mark.parametrize('s', [0.9, 1.5, 2.0])
def test_zoom_multiplies_the_flow(s):
    gt = np.broadcast_to(np.array([1.25, -0.75]), (1, H, W, 2)).copy()
    _, _, out = _run(AR.geometry(H, W, s=s), gt)
    assert np.abs(out - s * gt).max() <= 1e-12


def test_rotation_rotates_the_vectors_by_minus_theta():
    u, v = 2.0, -1.0
    gt = np.broadcast_to(np.array([-v, -u]), (1, H, W, 2)).copy()          # PWC-Net's order: (-v, -u)
    deg = 12.0
    _, _, out = _run(AR.geometry(H, W, deg=deg), gt)
    th = -math.radians(deg)
    u2, v2 = math.cos(th) * u - math.sin(th) * v, math.sin(th) * u + math.cos(th) * v
    assert np.abs(out[0, ..., 0] + v2).max() <= 1e-12 and np.abs(out[0, ..., 1] + u2).max() <= 1e-12


def test_relative_translation_adds_to_the_flow():
    gt = _smooth(1, H, W, 2, 2.0, 1)
    trx, try_ = 1.5, -0.75
    _, _, out = _run(AR.geometry(H, W, t_r=(trx, try_)), gt)
    assert np.abs(out[0, ..., 0] - (gt[0, ..., 0] + try_)).max() <= 1e-12
    assert np.abs(out[0, ..., 1] - (gt[0, ..., 1] + trx)).max() <= 1e-12


def test_frames_follow_their_maps():
    """frame 1 samples at T1(p), frame 2 at T2(p) = T1(Tr(p)): with T1 a translation and Tr another, frame 2 is moved by both."""
    img = np.clip(_smooth(1, H, W, 3, 0.2, 2), -0.5, 0.5)
    t1, t2 = AR.geometry(H, W, t=(3.0, 2.0), t_r=(-1.0, 4.0))
    o1, o2, _ = AR.augment(img, img, np.zeros((1, H, W, 2)), AR.row(t1, t2)[None])
    y, x = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing='ij')
    # no photometric change: (v + 0.5) - 0.5 in fp64
    assert np.abs(o1[0] - AR.bilinear(img[0], x + 3, y + 2)).max() <= 1e-15
    assert np.abs(o2[0] - AR.bilinear(img[0], x + 2, y + 6)).max() <= 1e-15


def test_photometric_chain_by_hand():
    v = np.array([[-0.3, 0.1, 0.45]])
    r = AR.row(*AR.geometry(4, 4), m=(2.0, 1.0, 0.5), contrast=0.5, beta=0.1, gamma=2.0, sigma=0.0)
    got = AR.photometric(v, r, 0.0)
    want = []
    for c, m in enumerate((2.0, 1.0, 0.5)):
        x = (v[0, c] + 0.5) * m
        x = 0.5 + 0.5 * (x - 0.5) + 0.1
        want.append(min(max(x, 0.0), 1.0) ** 2 - 0.5)
    assert np.allclose(got[0], want, rtol=0, atol=1e-15)
    # noise: added after gamma, then clamped
    n = np.array([[1.0, -2.0, 50.0]])
    r[24] = 0.01
    got = AR.photometric(v, r, n)
    assert np.allclose(got[0], np.minimum(np.array(want) + 0.5 + 0.01 * n[0], 1.0) - 0.5, rtol=0, atol=1e-15)


def test_noise_is_standard_normal_and_per_frame():
    a, b = AR.noise(12345, 0, 64, 96), AR.noise(12345, 1, 64, 96)
    assert abs(a.mean()) < 0.02 and abs(a.std() - 1) < 0.02 and abs(np.corrcoef(a.ravel(), b.ravel())[0, 1]) < 0.02


# ------------------------------------------------------------------------------------------------ the draws
def test_accepted_draws_keep_every_corner_inside():
    Hd, Wd, seed = 384, 640, 8964
    attempts = []
    for g in range(600):
        r = AR.sample_params({}, Hd, Wd, g, 7, seed)
        att = int(r[26])
        assert att < 64
        attempts.append(att)
        for m in (r[0:6], r[6:12]):
            assert AR.corners_inside(list(m), Hd, Wd)
        # T2^-1 o T2 = identity
        for x, y in ((0.0, 0.0), (639.0, 383.0), (17.5, 201.25)):
            qx, qy = AR.apply(r[6:12], x, y)
            bx, by = AR.apply(r[12:18], qx, qy)
            assert abs(bx - x) <= 1e-9 and abs(by - y) <= 1e-9
        assert 0.5 <= r[18:21].min() and r[18:21].max() <= 2.0 and 0.2 <= r[21] <= 1.4 and 0.7 <= r[23] <= 1.5 and 0 <= r[24] <= 0.04
    rate = len(attempts) / float(sum(a + 1 for a in attempts))
    print('MEASURED acceptance rate of the default geometry draws: %.3f' % rate)
    assert 0.26 <= rate <= 0.38            # 32 % by a 200k-draw model


def test_the_fallback_is_the_identity():
    r = AR.sample_params({'translate': (0.6, 0.7)}, 48, 80, 3, 0, 1)        # every T1 leaves the frame
    assert r[26] == 64
    assert list(r[0:18]) == [1, 0, 0, 0, 1, 0] * 3


def test_draws_use_their_own_counters():
    """attempt a draws k = 8a..8a+7; the photometric draws k = 512..520: a different step, sample or seed gives other draws."""
    base = AR.sample_params({}, 384, 640, 5, 3, 11)
    for g, t, seed in ((6, 3, 11), (5, 4, 11), (5, 3, 12)):
        assert not np.array_equal(AR.sample_params({}, 384, 640, g, t, seed), base)
    assert np.array_equal(AR.params({}, 3, 384, 640, 5, 3, 11)[0], base)


# ------------------------------------------------------------------------------------------------ C ABI
def test_struct_and_row_match_the_header(tmp_path):
    hdr = open(os.path.join(ROOT, 'include', 'cis_b200.h')).read()
    assert int(re.search(r'#define CIS_FLOW_AUG_ROW (\d+)', hdr).group(1)) == _lib.FLOW_AUG_ROW == AR.ROW
    r = flow_aug_ranges()
    for k, v in AUG_RANGES.items():
        assert np.allclose(np.float32(getattr(r, k) if not isinstance(v, tuple) else list(getattr(r, k))), np.float32(v))
        assert np.allclose(np.float32(v), np.float32(AR.DEFAULTS[k]))
    with pytest.raises(ValueError):
        flow_aug_ranges(zoom=(1, 2))
    if shutil.which('gcc') is None:
        pytest.skip('no gcc')
    src = tmp_path / 'sz.c'
    src.write_text('#include "%s"\n#include <stdio.h>\n#include <stddef.h>\nint main(){printf("%%zu %%zu %%zu %%zu\\n", sizeof(CisFlowAug), '
                   'offsetof(CisFlowAug, brightness), offsetof(CisFlowAug, gamma), offsetof(CisFlowAug, noise));return 0;}\n'
                   % os.path.join(ROOT, 'include', 'cis_b200.h'))
    exe = tmp_path / 'sz'
    subprocess.check_call(['gcc', str(src), '-o', str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(_lib.CisFlowAug), _lib.CisFlowAug.brightness.offset, _lib.CisFlowAug.gamma.offset, _lib.CisFlowAug.noise.offset]


def _bad_args():
    """(entry point, args) pairs that must be rejected before any launch; buffers are fake non-null addresses."""
    ok = flow_aug_ranges()
    p, odd = 1 << 20, (1 << 20) + 4
    aug = [('cis_flow_aug_params', (C.byref(ok), B, h, w, off, p, 1, p)) for B, h, w, off in
           ((0, 8, 8, 0), (65536, 8, 8, 0), (1, 1, 8, 0), (1, 8, 1, 0), (1, 8, 8, -1))]
    aug += [('cis_flow_aug_params', (C.byref(ok), 1, 8, 8, 0, None, 1, p)), ('cis_flow_aug_params', (C.byref(ok), 1, 8, 8, 0, p, 1, None)),
            ('cis_flow_aug_params', (None, 1, 8, 8, 0, p, 1, p))]
    for k, v in (('scale', (0.0, 1.0)), ('color', (2.0, 1.0)), ('gamma', (1.5, 0.7)), ('rel_scale', (-1.0, 1.0))):
        aug.append(('cis_flow_aug_params', (C.byref(flow_aug_ranges(**{k: v})), 1, 8, 8, 0, p, 1, p)))
    ok_aug = (p, p, p, p, 1, 8, 8, p, p, p)
    for i, v in ((4, 0), (4, 65536), (5, 1), (6, 1), (0, None), (1, None), (2, None), (3, None), (7, None), (8, None), (9, None),
                 (2, odd), (9, odd), (5, 20000), ):
        a = list(ok_aug)
        a[i] = v
        if i == 5 and v == 20000:
            a[6] = 20000                                # 6 H W >= 2^31
        aug.append(('cis_flow_augment', tuple(a)))
    return aug


def test_argument_errors_are_rejected_without_a_launch():
    lib = _lib.load()
    for name, args in _bad_args():
        rc = getattr(lib, name)(*args, None)
        assert rc == 1, (name, args)                     # CIS_ERR_BAD_ARG
        assert name.encode() in lib.cis_last_error()


# ------------------------------------------------------------------------------------------------ the training graph
def _digest(g):
    import plan_digest
    return plan_digest.digest([('fwd', g.fwd), ('bwd', g.bwd), ('adam', g.adam), ('pack', g.pack)])


@pytest.mark.parametrize('in_hw', [None, (384, 640)])
def test_augmented_step_is_the_plain_step_on_the_augmented_buffers(in_hw):
    import plan_digest
    B, Hg, Wg = 2, 128, 128
    with plan_digest.filled_uninitialized():
        off = FlowTrainGraph(Hg, Wg, B, device='cpu', in_hw=in_hw)
        on = FlowTrainGraph(Hg, Wg, B, device='cpu', in_hw=in_hw, augment=True, sample_offset=6)
        assert _digest(on) == _digest(off)          # the same launches, the step's inputs in the first three storages it references
    ih, iw = in_hw or (Hg, Wg)
    assert not off.aug.ops and not off.copy_in.ops and off.batch == off.inputs
    assert [op[2] for op in on.aug.ops] == ['cis_flow_aug_params', 'cis_flow_augment']
    pa, ag = on.aug.ops[0][1], on.aug.ops[1][1]
    assert pa[1:] == (B, ih, iw, 6, on.step_state.data_ptr(), on.aug_seed, on.aug_params.data_ptr())
    assert ag == tuple(t.data_ptr() for t in on.inputs) + (on.aug_params.data_ptr(), B, ih, iw) + tuple(t.data_ptr() for t in on.batch)
    # the step never reads the upload itself: only through the augmented buffers
    up = {t.data_ptr() for t in on.inputs}
    for plan in (on.fwd, on.bwd, on.adam, on.pack):
        for op in plan.ops:
            args = op[1] if isinstance(op[1], tuple) else ()
            assert not up & {a for a in args if isinstance(a, int)}, op[2]
    # the launch count of a step: two more
    assert on.launches_per_step() == off.launches_per_step() + 2


def test_forward_copies_and_train_step_augments(monkeypatch):
    g = FlowTrainGraph(128, 128, 2, device='cpu', augment=True)
    # forward(): three copies of the upload, no augmentation
    assert [op[2] for op in g.copy_in.ops] == ['copy'] * 3 and all(op[0] is None for op in g.copy_in.ops)
    for t in g.inputs:
        t.copy_(torch.randn(t.shape))
    for op in g.copy_in.ops:
        op[1]()
    assert all(torch.equal(a, b) for a, b in zip(g.batch, g.inputs))
    calls = []
    monkeypatch.setattr(g, '_ensure_packed', lambda: None)
    for name in ('copy_in', 'aug', 'fwd', 'bwd', 'adam', 'pack'):
        monkeypatch.setattr(getattr(g, name), 'run', lambda n=name: calls.append(n))
    g.forward()
    assert calls == ['copy_in', 'fwd']
    del calls[:]
    g.train_step()
    assert calls == ['aug', 'fwd', 'bwd', 'adam', 'pack']


def test_augment_is_refused_for_the_unsupervised_loss():
    with pytest.raises(ValueError):
        FlowTrainGraph(128, 128, 1, device='cpu', loss='unsupervised', augment=True)
    with pytest.raises(ValueError):
        FlowTrainGraph(128, 128, 1, device='cpu', augment=True, sample_offset=-1)
    FlowTrainGraph(128, 128, 1, device='cpu', loss='robust', augment=True, aug_ranges=flow_aug_ranges(noise=(0.0, 0.0)))


# ------------------------------------------------------------------------------------------------ train_flow.py
def test_train_flow_aug_usage_and_flag_dump(monkeypatch, tmp_path, capsys):
    sys.path.insert(0, ROOT)
    import train_flow as TF
    from unsupervised_detection_b200.common_flags import FLAGS, FLAG_NAMES
    from unsupervised_detection_b200.models import flow_learner
    assert 'flow_aug' in TF.TRAIN_FLOW_FLAGS and not set(TF.TRAIN_FLOW_FLAGS) & set(FLAG_NAMES)
    root = make_chairs_tree(tmp_path / 'chairs', n=2, labels=[1, 2])
    seen = []
    monkeypatch.setattr(flow_learner.FlowLearner, 'train_flow', lambda self, cfg: seen.append((cfg.flow_loss, cfg.flow_aug)))
    ck = '--checkpoint_dir=%s' % (tmp_path / 'ck')

    def main(*args):
        FLAGS.unparse_flags()
        TF.main(['train_flow.py', ck, '--dataset=FLYINGCHAIRS', '--root_dir=' + root] + list(args))
    try:
        main()
        assert "'flow_aug': False" in capsys.readouterr().out
        main('--flow_aug')
        assert "'flow_aug': True" in capsys.readouterr().out
        main('--flow_aug', '--flow_loss=robust')
        with pytest.raises(SystemExit) as e:
            main('--flow_aug', '--flow_loss=unsupervised')
        assert '--flow_aug' in str(e.value)
    finally:
        FLAGS.unparse_flags()
    assert seen == [('multiscale', False), ('multiscale', True), ('robust', True)]
