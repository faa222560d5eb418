"""Canonical text digest of launch plans, for checking that a change to the plan builders leaves every launch as it was.

One line per op: entry point, lane, flops and the arguments -- scalars by value, ctypes descriptors (CisConv, CisWgrad, CisSrc[],
int32[]) field by field, and every pointer as (storage k, storage bytes, byte offset) with storages numbered by first appearance.
A pointer is resolved by interval search over the untyped storages of the live CPU tensors, so plans must be built with
device='cpu'; a pointer into no storage is an error.  The job tables of cis_param_multi are decoded (their pointers become canonical
too), and every other referenced storage is listed with the SHA-256 of its bytes (kmap / nmap tables, parameters).  Uninitialised
allocations are filled with a fixed value while the plans are built, so buffers from torch.empty hash the same on every build.

    python tests/plan_digest.py OUT.txt      # every plan of the step graphs and the functional runners; CIS_* switches apply
"""
import bisect
import contextlib
import ctypes as C
import gc
import hashlib
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from unsupervised_detection_b200 import _lib  # noqa: E402


class _Storages(object):
    """Live CPU storages by address; numbers them in order of first reference."""

    def __init__(self):
        spans = {}
        for o in gc.get_objects():
            if type(o) in (torch.Tensor, torch.nn.Parameter) and o.device.type == 'cpu':
                st = o.untyped_storage()
                if st.nbytes():
                    spans[st.data_ptr()] = st
        self.starts = sorted(spans)
        self.st = [spans[p] for p in self.starts]
        self.order = []           # storage indices in first-reference order
        self.num = {}
        self.decoded = set()      # storages shown decoded (job tables) instead of hashed

    def find(self, p):
        i = bisect.bisect_right(self.starts, p) - 1
        if i < 0 or p >= self.starts[i] + self.st[i].nbytes():
            raise ValueError('pointer 0x%x is in no live CPU storage' % p)
        if i not in self.num:
            self.num[i] = len(self.order)
            self.order.append(i)
        return i

    def ptr(self, p):
        if not p:
            return 'null'
        i = self.find(p)
        return '(s%d,%d,+%d)' % (self.num[i], self.st[i].nbytes(), p - self.starts[i])

    def bytes_of(self, i):
        st = self.st[i]
        return torch.empty(0, dtype=torch.uint8).set_(st, 0, (st.nbytes(),)).numpy().tobytes()

    def raw(self, p, n):
        i = self.find(p)
        off = p - self.starts[i]
        return self.bytes_of(i)[off:off + n]

    def listing(self):
        out = []
        for i in self.order:
            h = 'decoded' if i in self.decoded else hashlib.sha256(self.bytes_of(i)).hexdigest()
            out.append('storage s%d %d %s' % (self.num[i], self.st[i].nbytes(), h))
        return out


def _value(v, ctype, S):
    if ctype is C.c_void_p:
        return S.ptr(v)
    if type(v).__name__ == 'CArgObject':
        v = v._obj
    if isinstance(v, C.Structure):
        return '{' + ' '.join('%s=%s' % (f, _value(getattr(v, f), t, S)) for f, t in v._fields_) + '}'
    if isinstance(v, C.Array):
        return '[' + ','.join(_value(x, v._type_, S) for x in v) + ']'
    if isinstance(v, float):
        return repr(v)
    return str(v)


def _param_jobs(args, S):
    """cis_param_multi(table, njobs, blocks): the job table read back from its storage, pointers canonical."""
    tab, njobs = args[0], args[1]
    i = S.find(tab)
    S.decoded.add(i)
    jobs = (_lib.CisParamJob * njobs).from_buffer_copy(S.raw(tab, njobs * C.sizeof(_lib.CisParamJob)))
    return [_value(j, None, S) for j in jobs]


def _op_line(op, S):
    fn, args, name, flops, lane = op
    if fn is None:
        return '%s lane=%d' % (name, lane)
    protos = _lib._PROTOS.get(name, [None] * len(args))
    vals = [_value(a, t, S) for a, t in zip(args, protos)]
    line = '%s lane=%d flops=%r %s' % (name, lane, flops, ' '.join(vals))
    if name == 'cis_param_multi':
        line += ' jobs=' + ' '.join(_param_jobs(args, S))
    return line


def digest(plans):
    """plans: [(label, Plan)] built on CPU tensors that are still alive -> list of lines (storages numbered across the plans)."""
    S = _Storages()
    out = []
    for label, plan in plans:
        out.append('# %s %s' % (label, plan.name))
        out += [_op_line(op, S) for op in plan.ops]
    return out + S.listing()


@contextlib.contextmanager
def filled_uninitialized():
    """torch.empty & co. fill new memory with NaN / the largest integer (torch's deterministic mode) instead of leaving it as found."""
    import torch.utils.deterministic as D
    prev = torch.are_deterministic_algorithms_enabled(), D.fill_uninitialized_memory
    torch.use_deterministic_algorithms(True)
    D.fill_uninitialized_memory = True
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev[0])
        D.fill_uninitialized_memory = prev[1]


def graph_plans(g):
    out = [('fwd', g.fwd), ('pack_pwc', g.pack_pwc), ('pack_gen', g.pack_gen), ('pack_rec', g.pack_rec)]
    for m in sorted(g.bwd):
        out += [('bwd' + m, g.bwd[m]), ('adam' + m, g.adam[m])]
    return out


def runner_plans(r):
    return [('fwd', r.bld.fwd), ('pack', r.pack), ('bwd', r.bwd)]


def _graph(*a, **k):
    from unsupervised_detection_b200.step_graph import CISGraph
    g = CISGraph(*a, device='cpu', **k)
    return g, graph_plans(g)


def _runner(cls, *a, **k):
    from unsupervised_detection_b200.models import functional as F
    r = getattr(F, cls)(*a, **k)
    r.ensure_backward()
    return r, runner_plans(r)


def _cases():
    ELU, LEAKY = _lib.ACT_ELU, _lib.ACT_LEAKY
    yield 'graph 64x96 b1 gb2', lambda: _graph(64, 96, 1, global_batch=2)
    yield 'graph 256x448 b4', lambda: _graph(256, 448, 4)
    small = dict(pwc_hw=(128, 192))
    yield 'graph pwc dense off', lambda: _graph(64, 96, 1, pwc_options={'use_dense_cx': False}, **small)
    yield 'graph pwc range 3', lambda: _graph(64, 96, 1, pwc_options={'search_range': 3}, **small)
    yield 'graph no pwc no train', lambda: _graph(64, 96, 1, with_pwc=False, train=False, **small)
    yield 'graph boxes', lambda: _graph(64, 96, 2, masks='boxes', box=(6, 32, 9, 48), sample_offset=2, **small)
    yield 'generator', lambda: _runner('_GeneratorRunner', 2, 64, 96, 'cpu', 'MaskNet')
    yield 'recover', lambda: _runner('_RecoverRunner', 2, 64, 96, 'cpu', 'FlownetS', 0.25)
    for opts in (None, {'use_dense_cx': False}, {'use_res_cx': False}, {'search_range': 2}):
        yield 'pwc %s' % (opts,), lambda o=opts: _runner('_PWCRunner', 1, 128, 192, 'cpu', 'pwcnet', trainable=True, options=o)
    for cin, spec, B, H, W in ((20, ('gen', 3, 16, 2, 1, ELU, None, None, 'Net/l'), 2, 37, 53),
                               (20, ('gen', 1, 16, 2, 1, ELU, None, None, 'Net/l'), 2, 37, 53),
                               (64, ('gen', 3, 32, 1, 1, ELU, 'nn2x', None, 'MaskNet/conv13_upsample'), 1, 16, 24),
                               (20, ('conv', 4, 8, 1, 1, LEAKY, 'bilinear', (9, 13), 'FlownetS/deconv5'), 1, 5, 7),
                               (64, ('conv', 3, 200, 1, 9, LEAKY, None, None, 'Net/l'), 2, 37, 53)):
        yield 'layer %s' % (spec,), lambda a=(B, H, W, cin, spec, 'cpu'): _runner('_LayerRunner', *a)


def main(path):
    with open(path, 'w') as f:
        for name, build in _cases():
            with filled_uninitialized():
                owner, plans = build()         # the owner keeps every buffer the plans point into alive
            f.write('## %s\n' % name)
            f.write('\n'.join(digest(plans)) + '\n')
            del owner, plans
            gc.collect()


if __name__ == '__main__':
    main(sys.argv[1])
