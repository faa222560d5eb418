"""Layer primitives of convolution_utils.py and preprocess_flow_batch (models/functional.py) without a GPU: every cell of the supported set
plans its forward and backward on CPU tensors, the test-side bilinear reference (tests/resize_ref.py) against hand-computed values, argument errors, the
kernel calls of the resizes and the flow standardisation (recorded, not run), and the two things this work must not move: the SASS of
the legacy fp32 resize kernels and the step graph's launch plan.  The numerical checks live in test_layer_api_gpu.py."""
import hashlib
import os
import re
import shutil
import subprocess
import sys

import pytest
import torch

import resize_ref
from oracle import tf_ops as T
from unsupervised_detection_b200 import _lib, engine
from unsupervised_detection_b200.models import functional as F
from unsupervised_detection_b200.models.utils import convolution_utils as CU
from unsupervised_detection_b200.models.utils import flow_utils as FU

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H, W = 37, 53


def _names(plan):
    return [op[2] for op in plan.ops if op[0] is not None]


@pytest.fixture
def stubbed(monkeypatch):
    """Plans are built for real but never replayed; kernel calls of the stand-alone ops are recorded."""
    calls = []
    monkeypatch.setattr(engine.Plan, 'run', lambda self, stream=None, lane_key=0: None)
    monkeypatch.setattr(F._lib, 'call', lambda name, *a: calls.append((name, a)))
    monkeypatch.setattr(F, '_check_cuda', lambda *t: None)
    monkeypatch.setattr(F, '_stream', lambda: 0)
    monkeypatch.setattr(F, '_RUNNERS', {})
    monkeypatch.setattr(F, '_POOLS', {})
    return calls


# ------------------------------------------------------------------------------------------------------------ planning
CELLS = ([(k, s, 1, bn) for k in range(1, 8) for s in (1, 2) for bn in (True, False)] +
         [(3, 1, r, bn) for r in (2, 3, 4, 8, 9, 16) for bn in (True, False)])


@pytest.mark.parametrize('cin,cout', [(3, 1), (20, 16), (64, 200)])
@pytest.mark.parametrize('k,stride,rate,bn', CELLS)
def test_every_cell_plans_forward_and_backward(k, stride, rate, bn, cin, cout):
    kind = 'gen' if bn else 'conv'
    r = F._LayerRunner(2, H, W, cin, (kind, k, cout, stride, rate, _lib.ACT_ELU if bn else _lib.ACT_LEAKY, None, None, 'Net/l'), 'cpu')
    assert tuple(r.outf.shape) == (2, -(-H // stride), -(-W // stride), cout)
    r.ensure_backward()
    names = _names(r.bwd)
    assert names[0] == 'cis_cast_f32_to_bf16' and names[-1] == 'cis_cast_bf16_to_f32'
    assert r.x8.grad_written.get('L') and r.x8.grad is not None                  # the data gradient reaches the input Act
    assert names.count('cis_conv_wgrad') == -(-cout // 128)                       # launches of at most 128 output channels
    want = ['Net/l/kernel', 'Net/l/bias', 'Net/l/gamma', 'Net/l/beta'] if bn else ['Net/l/weights', 'Net/l/biases']
    assert r.param_names() == want
    shapes = [e[1] for e in r.store.entries]
    assert shapes[0] == (k, k, cin, cout) and all(s == (cout,) for s in shapes[1:])
    # tapless output parities (k = 1, stride 2) zero the input gradient once, before the parity launches
    tapless = stride == 2 and k == 1
    assert names.count('cis_add_slice') == (1 if tapless else 0)
    if tapless:
        assert names.index('cis_add_slice') < names.index('cis_conv_igemm')
        z = next(op[1] for op in r.bwd.ops if op[2] == 'cis_add_slice')
        g = r.x8.grad
        assert z[:3] == (g.ptr, g.pitch, g.c_off) and z[6:] == (2 * H * W, g.C8 // 8, 0, 0)
        assert sum(1 for pk in r.layer.dgrad_packs if not pk['taps']) == 3
    assert not any(op[2].startswith('cis_pack_weights') and op[1][2] == 0 for op in r.pack.ops)   # no pack of an empty tap set


def test_tapless_parity_accumulates_without_zeroing():
    """A second reader of the same Act accumulates: the tapless parity leaves the gradient untouched, so nothing is zeroed."""
    store, bld = engine.ParamStore('cpu'), engine.Builder('cpu')
    L1 = engine.ConvLayer(store, 'a', 1, 8, 16, 2, tag='L', wname='weights', bname='biases')
    L2 = engine.ConvLayer(store, 'b', 3, 8, 16, 1, tag='L', wname='weights', bname='biases')
    store.finalize(False)
    x = bld.new_act(1, H, W, 8, dep={'L'})
    y1 = bld.conv(L1, [x])
    y2 = bld.conv(L2, [x])
    bp = bld.build_backward('L', [y2, y1])           # y1's backward runs last: x.grad already holds L2's data gradient
    assert 'cis_add_slice' not in _names(bp) and x.grad_written['L']


def test_pre_ops_plan_their_backward():
    r = F._LayerRunner(1, 16, 24, 64, ('gen', 3, 32, 1, 1, _lib.ACT_ELU, 'nn2x', None, 'MaskNet/conv13_upsample'), 'cpu')
    assert tuple(r.outf.shape) == (1, 32, 48, 32)
    r.ensure_backward()
    assert 'cis_upsample_nn2x' in _names(r.bld.fwd) and 'cis_upsample_nn2x_bwd' in _names(r.bwd)
    r = F._LayerRunner(1, 5, 7, 20, ('conv', 4, 8, 1, 1, _lib.ACT_LEAKY, 'bilinear', (9, 13), 'FlownetS/deconv5'), 'cpu')
    assert tuple(r.outf.shape) == (1, 9, 13, 8)
    r.ensure_backward()
    assert 'cis_resize_bilinear_bf16' in _names(r.bld.fwd) and 'cis_resize_bilinear_bf16_bwd' in _names(r.bwd)
    assert r.x8.grad_written.get('L')


def test_layer_calls_through_the_public_module(stubbed):
    x = torch.zeros(2, H, W, 20)
    p = {'G/c/kernel': torch.zeros(3, 3, 20, 16), 'G/c/bias': torch.zeros(16), 'G/c/gamma': torch.ones(16), 'G/c/beta': torch.zeros(16)}
    y = CU.gen_conv(x, 16, 3, 2, name='G/c', params=p)
    assert tuple(y.shape) == (2, 19, 27, 16) and y.grad_fn is None and not F._POOLS
    (r,) = F._RUNNERS.values()
    assert r.layer.act == _lib.ACT_ELU and r.layer.bn and r.bwd is None
    x.requires_grad_(True)
    y = CU.gen_conv(x, 16, 3, 2, name='G/c', params=p)
    assert y.grad_fn is not None and len(F._POOLS) == 1
    # a callable that is not one of the fused three runs on an identity-activation conv and is applied afterwards
    seen = []
    CU.gen_conv(x.detach(), 16, 3, 2, name='G/c', params=p, activation=lambda t: seen.append(t) or t)
    assert len(seen) == 1 and F._RUNNERS[[k for k in F._RUNNERS if k[-5] == _lib.ACT_NONE][0]].layer.act == _lib.ACT_NONE
    q = {'R/f/weights': torch.zeros(3, 3, 20, 2), 'R/f/biases': torch.zeros(2)}
    y = CU.conv(x.detach(), 'R/f', [3, 3, 20, 2], 1, activation=CU.identity, params=q)
    assert tuple(y.shape) == (2, H, W, 2)
    y = CU.deconv(x.detach(), [74, 106], 'R/f', [3, 3, 20, 2], params=q)
    assert tuple(y.shape) == (2, 74, 106, 2)
    d = {'G/u/kernel': torch.zeros(3, 3, 20, 8), 'G/u/bias': torch.zeros(8), 'G/u/gamma': torch.ones(8), 'G/u/beta': torch.zeros(8)}
    assert tuple(CU.gen_deconv(x.detach(), 8, name='G/u', params=d).shape) == (2, 2 * H, 2 * W, 8)


def test_unsupported_arguments_raise(stubbed):
    x = torch.zeros(1, 8, 8, 4)
    p = {'c/kernel': torch.zeros(3, 3, 4, 8), 'c/bias': torch.zeros(8), 'c/gamma': torch.zeros(8), 'c/beta': torch.zeros(8)}
    for kw in (dict(ksize=8), dict(ksize=0), dict(ksize=[3, 5]), dict(ksize=3, stride=3), dict(ksize=3, rate=17),
               dict(ksize=3, stride=2, rate=2), dict(ksize=3, padding='VALID')):
        kw.setdefault('ksize', 3)
        with pytest.raises(NotImplementedError, match='supported set'):
            CU.gen_conv(x, 8, name='c', params=p, **kw)
    with pytest.raises(NotImplementedError, match='non-square'):
        CU.conv(x, 'c', [3, 5, 4, 8], 1)
    with pytest.raises(ValueError, match='shape\\[2\\]'):
        CU.conv(x, 'c', [3, 3, 5, 8], 1)
    with pytest.raises(ValueError, match='shape\\[2\\]'):
        CU.deconv(x, [16, 16], 'c', [3, 3, 5, 8])
    with pytest.raises(KeyError, match='c/beta'):
        CU.gen_conv(x, 8, 3, name='c', params={k: v for k, v in p.items() if k != 'c/beta'})
    with pytest.raises(ValueError, match='c/kernel'):
        CU.gen_conv(x, 8, 3, name='c', params=dict(p, **{'c/kernel': torch.zeros(3, 3, 8, 4)}))
    with pytest.raises(ValueError, match='size'):
        CU.resize_bilinear(x, [0, 4])
    with pytest.raises(ValueError, match='2\\]'):
        FU.preprocess_flow_batch(torch.zeros(1, 4, 4, 3))


def test_cpu_tensors_have_no_fallback():
    for call in (lambda: CU.resize_bilinear(torch.zeros(1, 4, 4, 2), [8, 8]), lambda: FU.preprocess_flow_batch(torch.zeros(1, 4, 4, 2)),
                 lambda: CU.gen_conv(torch.zeros(1, 4, 4, 2), 4, 3, name='c', params={})):
        with pytest.raises(RuntimeError, match='no CPU fallback'):
            call()


# --------------------------------------------------------------------------------------------------- resizes + flow kernels
def test_resize_calls_record_method_and_align_corners(stubbed):
    x = torch.zeros(2, 5, 7, 3)
    CU.resize(x)                                                            # default: bilinear, align_corners=True, x2
    CU.resize(x, func=CU.resize_nearest_neighbor, to_shape=[3, 4], align_corners=False)
    CU.resize_bilinear(x, [11, 2])
    CU.resize_nearest_neighbor(x, (1, 9), align_corners=True)
    got = [(n, a[1:5], a[6:10]) for n, a in stubbed]
    assert got == [('cis_resize_f32', (2, 5, 7, 3), (10, 14, _lib.RESIZE_BILINEAR, 1)),
                   ('cis_resize_f32', (2, 5, 7, 3), (3, 4, _lib.RESIZE_NEAREST, 0)),
                   ('cis_resize_f32', (2, 5, 7, 3), (11, 2, _lib.RESIZE_BILINEAR, 0)),
                   ('cis_resize_f32', (2, 5, 7, 3), (1, 9, _lib.RESIZE_NEAREST, 1))]
    seen = []
    CU.resize(x, scale=1.5, func=lambda t, size, align_corners: seen.append((size, align_corners)))
    assert seen == [([7, 10], True)]


def test_resize_backward_call(stubbed):
    x = torch.zeros(1, 5, 7, 3, requires_grad=True)
    y = CU.resize_nearest_neighbor(x, [9, 4], align_corners=True)
    y.backward(torch.zeros(1, 9, 4, 3))
    name, a = stubbed[-1]
    assert name == 'cis_resize_f32_bwd' and a[1:7] == (1, 9, 4, 3, 5, 7) and a[8:10] == (_lib.RESIZE_NEAREST, 1)
    assert x.grad.shape == x.shape


def test_flow_standardisation_calls(stubbed):
    f = torch.zeros(3, 6, 10, 2, requires_grad=True)
    y = FU.preprocess_flow_batch(f)
    y.backward(torch.zeros_like(y))
    assert [n for n, _ in stubbed] == ['cis_flow_stats', 'cis_flow_standardize', 'cis_flow_standardize_bwd']
    (_, st), (_, fw), (_, bw) = stubbed
    assert st[1:3] == (3, 60) and fw[1] == st[3] and fw[2:4] == (3, 60)
    assert bw[2] == st[3] and bw[3:5] == (3, 60)


def test_new_entry_points_are_declared_in_the_header():
    hdr = open(os.path.join(ROOT, 'include', 'cis_b200.h')).read()
    for name in ('cis_resize_f32', 'cis_resize_f32_bwd', 'cis_flow_standardize', 'cis_flow_standardize_bwd'):
        assert name in _lib.EXPORTS and re.search(r'\bint %s\(' % name, hdr)
        n_args = len(re.search(r'\bint %s\(([^)]*)\)' % name, hdr).group(1).split(','))
        assert n_args == len(_lib._PROTOS[name]) + 1, name                # + the stream


# ---------------------------------------------------------------------------------------------------------- reference
def test_reference_align_corners_bilinear_hand_values():
    x = torch.tensor([1.0, 3.0], dtype=torch.float64).view(1, 2, 1, 1)
    assert resize_ref.resize_bilinear(x, 3, 1, True).flatten().tolist() == [1.0, 2.0, 3.0]        # the exact midpoint
    y = torch.arange(12, dtype=torch.float64).view(1, 3, 4, 1)
    assert resize_ref.resize_bilinear(y, 1, 1, True).flatten().tolist() == [0.0]                   # out = 1: scale 0
    assert resize_ref.resize_bilinear(y, 1, 4, True).flatten().tolist() == [0.0, 1.0, 2.0, 3.0]
    # downscale 4 -> 3 columns: scale 1.5 -> src 0, 1.5, 3; 3 -> 2 rows: scale 2 -> src 0, 2
    assert resize_ref.resize_bilinear(y, 2, 3, True).flatten().tolist() == [0.0, 1.5, 3.0, 8.0, 9.5, 11.0]
    # legacy (align_corners=False): step in/out, 2 -> 4 samples reads src 0, 0.5, 1, 1.5 -> the last one clamps to the edge
    assert resize_ref.resize_bilinear(x, 4, 1, False).flatten().tolist() == [1.0, 2.0, 3.0, 3.0]


# --------------------------------------------------------------------------------------------------- things that must not move
PARENT_SASS = {  # sha256 of the instruction text (cuobjdump -sass, addresses stripped) of the parent's kernels, CUDA 12.9
    '_ZN3cis26resize_bilinear_f32_kernelILb0EEEvPKfiiiiPfiif': '5a528314e62ecae830c5986231f637bc6c2304a1c89131b10c9e79d27cb55fee',
    '_ZN3cis20resize_nn_f32_kernelILb0EEEvPKfiiiiPfii': 'a90ea362d5a6bb71124acb077a54e2d263ccc081b099d7d742c2a2d17aef246f',
}
PARENT_PLAN_REPORT = 'be7635be69ede13dc8f149930ebffcff9f80b32fb053193405b108584436bb48'


def _sass_functions(path):
    out, cur = {}, None
    for line in subprocess.check_output([_cuobjdump(), '-sass', path], text=True).splitlines():
        if line.strip().startswith('Function :'):
            cur = out.setdefault(line.split(':', 1)[1].strip(), [])
            continue
        m = re.match(r'\s*/\*[0-9a-f]{4}\*/\s*(.*?);', line)
        if m and cur is not None:
            cur.append(m.group(1).strip())
    return out


def _cuobjdump():
    exe = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(exe):
        pytest.skip('cuobjdump not installed')
    return exe


def test_legacy_fp32_resize_kernels_compile_to_the_parents_sass():
    """The align_corners = false instances of the templated kernels are instruction for instruction what the step graph ran before."""
    if subprocess.run([_cuobjdump(), '--version'], capture_output=True, text=True).stdout.find('12.9') < 0:
        pytest.skip('the recorded SASS is that of CUDA 12.9')
    fns = _sass_functions(_lib.LIB_PATH)
    for name, digest in PARENT_SASS.items():
        assert hashlib.sha256('\n'.join(fns[name]).encode()).hexdigest() == digest, name


def test_step_graph_launch_plan_is_unchanged():
    env = {k: v for k, v in os.environ.items() if not k.startswith('CIS_')}
    out = subprocess.check_output([sys.executable, os.path.join(ROOT, 'tools', 'plan_report.py')], env=env, cwd=ROOT)
    assert hashlib.sha256(out).hexdigest() == PARENT_PLAN_REPORT


def test_halo_wgrad_fit_counts_both_gradient_tiles():
    """Cout > 64 runs two MMA warpgroups, each with its own 8x8-pixel gradient tile per stage: a rate-9 3x3 layer (26x26 halo) then no
    longer fits two stages in shared memory and takes the TMA weight-gradient kernel; Cout <= 64 (one tile) still fits."""
    taps = [(a * 9 - 9, b * 9 - 9) for a in range(3) for b in range(3)]
    assert not engine.wgrad_halo_fits(taps, 200, 1) and not engine.wgrad_halo_fits(taps, 72, 1)
    assert engine.wgrad_halo_fits(taps, 64, 1)
    r = F._LayerRunner(1, H, W, 64, ('gen', 3, 200, 1, 9, _lib.ACT_ELU, None, None, 'Net/l'), 'cpu')
    r.ensure_backward()
    assert not r.layer.wg_halo
    wg = [op[1][0]._obj for op in r.bwd.ops if op[2] == 'cis_conv_wgrad']
    assert [w.tma for w in wg] == [1, 1]
