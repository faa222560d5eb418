"""Every convolution launch of a launch plan, checked on its own against an fp64 reference of the same operation.

Recorder
    `recorded(monkeypatch)` wraps Builder.conv, _conv_bwd, conv_transpose and _conv_transpose_bwd while graphs are built and notes which
    cis_conv_igemm / cis_conv_wgrad op tuples each call appended to its plan, with the Acts and the layer involved.  Backward plans extend
    plans with the same tuple objects, so op identity survives into the step's bwd plans.  Every such op is attributed to exactly one check:
    a forward launch group (one launch, or the four output-parity launches of a transposed conv), the data-gradient launch group of one
    layer call (one launch, four parity launches or one grouped launch), or one weight-gradient launch of one layer call.

Executor
    `Walker.run(plan)` replays a plan's ops in order on the current stream, calling fn(*args, stream) exactly as Plan.run(stream=...) does
    (both lanes serialised on one stream, a legal order of the plan).  Before the first op of a check it snapshots what the launch reads --
    the real channels of every source, the output gradient G as it is at that moment (after cis_dact_colsum rewrote it), the whole
    destination buffer -- and after the last op it synchronises and compares.  Weight gradients are compared after the plan's finalize
    (cis_param_multi): the stored gradient of a layer against the fp64 sum over its calls.  Every other op runs unchecked.

References (torch float64 on the device)
    Each reference is computed from the bf16 values the launch actually read, so errors do not compound from layer to layer.  Weights are
    bf16(w_eff) (the layer's own folded buffer for BN layers, the fp32 master otherwise).

Per-element bound, no normalisation by the tensor maximum:

    |got - ref| <= e_out |ref| + gamma S + delta

    S is the same fp64 operation on absolute values (sum |a||w| for a forward element, sum |g||w| for a data gradient, sum |g||a| for a
    weight gradient, sum |g| for a bias gradient) plus the absolute values of the bias, residual and accumulate operands.

    e_out = 2^-8 for bf16 stores (round to nearest with an 8-bit significand: |bf16(v) - v| <= 2^-8 |v|), 0 for fp32 outputs.

    gamma.  The products of two bf16 values are exact in fp32.  What remains is the summation: for any summation tree in which a term goes
    through at most n additions, the first-order error is <= n u sum|term|.  u = 2^-23 covers an fp32 addition that truncates instead of
    rounding (the tensor cores align addends to the largest exponent and truncate).  A term goes through
      - the additions of its CTA's accumulator: at most the terms one split of the K loop owns (halo kernel: taps x 64 channels per
        64-channel chunk; gather kernel: 64 per K block; weight gradient: 64 pixels per reduction block),
      - the split-K partial sums (finish kernel) or the un-pack's fixed-order sum of the private slices of every split and call,
      - four epilogue additions (bias, accumulate or fp32 residual, skip).
    So gamma = (n_cta + n_partials + 4) 2^-23, times (1 + 2^-7) for bf16 stores (rounding the already perturbed value).  Bias gradients:
    n = pixels per column-sum block + blocks of every call.  The BN chain rule adds its own 32-lane fixed-order sum over the kernel rows.

    delta.  ELU computes exp through ex2.approx: relative error <= 2^-22 on e^x <= 1, plus the rounding of x log2(e) (<= 2^-24 / e after
    the exp) and of the final "- 1" (<= 2^-24): <= 3.7e-7 absolute, so delta = 2^-21 for ELU layers.  The mask epilogue sigma((x0 - x1)/10)
    adds __expf and a division: delta = 2^-20 on top of (gamma S0 + gamma S1) / 40 (sigma(z/10) is 1/40-Lipschitz).  Otherwise
    delta = 2^-100, a floor that keeps 0/0 out of the ratio.

Stray writes: after each checked launch, every element of the destination buffer outside the launch's rows x [out_coff, out_coff+out_ch)
must be bit-identical to its snapshot, and the padding channels inside the window must be exactly 0 (a NaN there would poison the next
layer: its zero weights do not mask it).

Negative controls (Walker(controls=True); a ratio > 1 means the bound rejected the corruption), made on the reference or on a copy of the
result, each for the first launch that qualifies:
  fwd.halo, fwd.gather, dgrad.parity_group, wgrad.<kind>: the reference without the centre tap of the weights;
  tile: one 16 x 8 tile of one channel of a bf16 output scaled by 1 + 2^-5, at the largest output;
  tile.partial: the same on the last 16 x 8 tile of a launch whose OW is not a multiple of 8 (a partial tile: columns past OW do not
    exist), at the sample and channel where that tile is largest;
  thin<t>.cin<c>: a compact thin-input launch (CisConv.thin = t) of a layer with c < t real input channels, against the reference without
    input channel c - 1 (the last real one; channels c .. t - 1 are the zero padding the format reads).
"""
import collections
import contextlib
import inspect

import torch
import torch.nn.functional as F

from oracle import tf_ops as T
from unsupervised_detection_b200 import _lib, engine as E
from unsupervised_detection_b200._lib import ACT_ELU, ACT_LEAKY

U = 2.0 ** -23
BN_RSQRT = float(torch.tensor(1.0 / (1.0 + 1e-3) ** 0.5, dtype=torch.float32))     # the fp32 constant of cis_bn_fold / cis_bn_chain
DELTA_FLOOR = 2.0 ** -100
DELTA_ELU = 2.0 ** -21
DELTA_MASK = 2.0 ** -20
E_BF16 = 2.0 ** -8


def smooth(B, H, W, C, amp, gen, div=16):
    lo = torch.randn(B, C, max(H // div, 2), max(W // div, 2), generator=gen)
    return (F.interpolate(lo, size=(H, W), mode='bicubic', align_corners=False) * amp).permute(0, 2, 3, 1).contiguous()


# ---------------------------------------------------------------------------------------------------------------- recorder
class Check(object):
    """kind: 'fwd' | 'dgrad' | 'wgrad'; ops: the op tuples of the check, in plan order; info: what the launches read and write."""

    def __init__(self, kind, layer, mode, call, ops, **info):
        self.kind, self.layer, self.mode, self.call, self.ops, self.info = kind, layer, mode, call, ops, info

    def descs(self):
        return [op[1][0]._obj for op in self.ops]

    def label(self):
        """Launch kind of the summary line."""
        d = self.descs()[0]
        if self.kind == 'wgrad':
            return 'wgrad.tr' if self.layer.transposed else 'wgrad.tma%d' % d.tma
        if self.layer.transposed:
            return 'fwd.tr_parity' if self.kind == 'fwd' else 'dgrad.tr'
        if self.kind == 'dgrad' and self.layer.stride == 2:
            return 'dgrad.parity_group' if d.nsub > 1 else 'dgrad.parity'
        return '%s.%s' % (self.kind, 'halo' if d.halo else 'gather')

    def __repr__(self):
        d = self.descs()[0]
        if self.kind == 'wgrad':
            geo = 'N%d %dx%d tma%d nh%d nwg%d splits%d Cout%d' % (d.N, d.OH, d.OW, d.tma, d.nh, d.nwg, d.splits, d.Cout)
        else:
            geo = 'N%d %dx%d halo%d MT%d nwg%d BN%d n_tiles%d splits%d nsub%d dil%d nsrc%d' % (
                d.N, d.OH, d.OW, d.halo, d.MT, d.nwg, d.BN, d.n_tiles, d.splits, d.nsub, d.dil, d.nsrc)
        return '%s %s mode=%s call=%d [%s] x%d' % (self.kind, self.layer.name, self.mode, self.call, geo, len(self.ops))


def persist_candidate(d):
    """The descriptor-side conditions of conv_halo_persist_kernel (csrc launch_halo); whether the weight set fits shared memory and the
    tile count are decided in the library at launch time."""
    return bool(d.halo and d.n_tiles == 1 and d.splits <= 1 and d.nph <= 1 and d.nsub <= 1 and d.dil == 1 and d.MT * d.BN <= 64
                and d.nwg <= 1)


class Recorder(object):
    def __init__(self):
        self.checks = []
        self.by_op = {}           # id(op tuple) -> Check
        self.fwd_calls = collections.Counter()

    def _add(self, ck):
        if not ck.ops:
            return
        for op in ck.ops:
            assert id(op) not in self.by_op, ('op attributed twice', ck)
            self.by_op[id(op)] = ck
        self.checks.append(ck)

    def install(self, mp):
        B = E.Builder
        o_conv, o_bwd, o_tr, o_trbwd = B.conv, B._conv_bwd, B.conv_transpose, B._conv_transpose_bwd
        rec = self

        def bind(fn, *a, **k):
            ba = inspect.signature(fn).bind(*a, **k)
            ba.apply_defaults()
            return ba.arguments

        def conv(*a, **k):
            ar = bind(o_conv, *a, **k)
            bld, layer = ar['self'], ar['layer']
            plan = ar['plan'] or bld.fwd
            n0, k0 = len(plan.ops), len(plan.keep)
            res = o_conv(*a, **k)
            keep = plan.keep[k0:]
            i = next(j for j, o in enumerate(keep) if o is layer)
            srcs, out, outf, addf, post_add = keep[i - 5:i]      # Builder.conv: plan.keep += [srcs, out, outf, addf, post_add, layer]
            ops = [op for op in plan.ops[n0:] if op[2] == 'cis_conv_igemm']
            call = rec.fwd_calls[id(layer)]
            rec.fwd_calls[id(layer)] += 1
            rec._add(Check('fwd', layer, None, call, ops, srcs=list(srcs), out=out, outf=outf, addf=addf, post_add=post_add,
                           mask_mode=ar['mode']))
            return res

        def conv_bwd(*a, **k):
            ar = bind(o_bwd, *a, **k)
            bp, mode, layer, srcs = ar['bp'], ar['mode'], ar['layer'], ar['srcs']
            n0 = len(bp.ops)
            res = o_bwd(*a, **k)
            new = bp.ops[n0:]
            gout = ar['grad_out'] if ar['grad_out'] is not None else ar['out']
            wg = [op for op in new if op[2] == 'cis_conv_wgrad']
            dg = [op for op in new if op[2] == 'cis_conv_igemm']
            if wg or dg:
                G = gout.get_grad()
            for op in wg:
                rec._add(Check('wgrad', layer, mode, ar['call'], [op], srcs=list(srcs), G=G))
            if dg:
                single = len(srcs) == 1 and srcs[0].n_mod == 0
                tgt = srcs[0].get_grad() if single else layer.dcat
                rec._add(Check('dgrad', layer, mode, ar['call'], dg, srcs=list(srcs), G=G, tgt=tgt))
            return res

        def conv_transpose(*a, **k):
            ar = bind(o_tr, *a, **k)
            bld, layer = ar['self'], ar['layer']
            plan = ar['plan'] or bld.fwd
            n0 = len(plan.ops)
            out = o_tr(*a, **k)
            ops = [op for op in plan.ops[n0:] if op[2] == 'cis_conv_igemm']
            call = rec.fwd_calls[id(layer)]
            rec.fwd_calls[id(layer)] += 1
            rec._add(Check('fwd', layer, None, call, ops, srcs=[ar['src']], out=out, outf=ar['outf'], addf=None, post_add=None,
                           mask_mode=0))
            return out

        def tr_bwd(*a, **k):
            ar = bind(o_trbwd, *a, **k)
            bp, mode, layer, src, out = ar['bp'], ar['mode'], ar['layer'], ar['src'], ar['out']
            n0 = len(bp.ops)
            res = o_trbwd(*a, **k)
            new = bp.ops[n0:]
            for op in new:
                if op[2] == 'cis_conv_wgrad':
                    rec._add(Check('wgrad', layer, mode, 0, [op], srcs=[src], G=out.get_grad()))
            dg = [op for op in new if op[2] == 'cis_conv_igemm']
            if dg:
                rec._add(Check('dgrad', layer, mode, 0, dg, srcs=[src], G=out.get_grad(), tgt=src.get_grad()))
            return res

        mp.setattr(B, 'conv', conv)
        mp.setattr(B, '_conv_bwd', conv_bwd)
        mp.setattr(B, 'conv_transpose', conv_transpose)
        mp.setattr(B, '_conv_transpose_bwd', tr_bwd)


@contextlib.contextmanager
def recorded(monkeypatch):
    """Graphs built inside the block are recorded; the Builder methods are restored when it ends."""
    rec = Recorder()
    with monkeypatch.context() as mp:
        rec.install(mp)
        yield rec


def conv_ops(plan):
    return [op for op in plan.ops if op[2] in ('cis_conv_igemm', 'cis_conv_wgrad')]


# ---------------------------------------------------------------------------------------------------------------- references
def _real(a, n):
    """Real channels of Act `a`, rows [:n], in original-channel order, as fp64."""
    pos = sorted((m, p) for p, m in enumerate(a.chanmap) if m >= 0)
    assert [m for m, _ in pos] == list(range(len(pos))), a.name
    idx = torch.tensor([a.c_off + p for _, p in pos], device=a.buf.device)
    return a.buf[:n].index_select(3, idx).double()


def _concat(srcs, n):
    """The virtual concat the launch reads: n rows, batch-broadcast (n_mod) sources repeated."""
    xs = []
    for s in srcs:
        x = _real(s, s.N)
        if s.n_mod:
            x = x[torch.arange(n, device=x.device) % s.n_mod]
        xs.append(x[:n])
    return torch.cat(xs, 3)


def _weights(L):
    k = L.k
    if L.bn:
        w = L.w_eff.view(k, k, L.cin, L.cout)
    else:
        w = L.store.view(L.wkey)
    return w.to(torch.bfloat16).double()


def _bias(L):
    return (L.b_eff[:L.cout] if L.bn else L.store.view(L.bkey)).double()


def _conv(L, x, w):
    if L.transposed:
        return T.conv2d_transpose_k4s2(x, w)
    return T.conv2d_same(x, w, L.stride, L.dil)


def _act(L, y):
    if L.act == ACT_ELU:
        return F.elu(y)
    if L.act == ACT_LEAKY:
        return F.leaky_relu(y, L.alpha)
    return y


def _conv_terms(d):
    """Additions one accumulator element goes through (see the module docstring)."""
    chunks = sum(d.src[i].chunks for i in range(d.nsrc))
    units, per = (-(-chunks // 8), d.ntaps * 64) if d.halo else (d.K_pad // 64, 64)
    sp = max(d.splits, 1)
    return per * (-(-units // sp)) + sp + 4


def _wgrad_terms(w):
    npix = w.N * w.OH * w.OW
    nkb = w.N * (-(-w.OH // 8)) * (-(-w.OW // 8)) if w.tma else -(-npix // 64)
    return 64 * (-(-nkb // w.splits))


def ratio(got, ref, S, e_out, gamma, delta):
    """max |got - ref| / (e_out |ref| + gamma S + delta); inf when got holds a non-finite value."""
    got = got.double()
    if not torch.isfinite(got).all():
        return float('inf')
    bound = e_out * ref.abs() + gamma * S + max(delta, DELTA_FLOOR)
    return float(((got - ref).abs() / bound).max())


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def stray(now, old, rows, c0, c1, pads):
    """'' or what is wrong: destination buffer `now` against its snapshot outside rows [:rows] x channels [c0, c1); padding channel
    positions `pads` (absolute) inside the window must be exactly 0."""
    a, b = _bits(now), _bits(old)
    if not torch.equal(a[rows:], b[rows:]):
        return 'rows >= %d changed' % rows
    if not torch.equal(a[:rows, ..., :c0], b[:rows, ..., :c0]) or not torch.equal(a[:rows, ..., c1:], b[:rows, ..., c1:]):
        return 'channels outside [%d, %d) changed' % (c0, c1)
    if pads:
        p = now[:rows].index_select(-1, torch.tensor(pads, device=now.device))
        if not bool((p == 0).all()):
            return 'padding channels %s not zero' % (pads,)
    return ''


class Walker(object):
    """Replays plans with every recorded conv launch checked.  results[label] = list of worst bound ratios; failures = messages;
    controls[name] = negative-control ratio (> 1: the bound rejected the corrupted comparison)."""

    def __init__(self, rec, controls=False, glue=None):
        self.rec = rec
        self.glue = glue            # a second checker for the ops it owns (glue_launch_ref.Glue), keyed on the entry point
        self.results = collections.defaultdict(list)
        self.persist = collections.Counter()
        self.failures = []
        self.controls = {} if controls else None
        self.wgrad = {}             # (layer id, mode) -> accumulated reference
        self.wgrad_seen = set()     # (layer id, mode, call) whose reference is in
        self.snap = None
        self.checked = 0            # conv launches checked
        self.launches = collections.Counter()     # label -> conv launches checked

    # ---- plan replay
    def run(self, plan):
        st = torch.cuda.current_stream().cuda_stream
        modes = set()
        if self.glue is not None:
            self.glue.start_plan(plan.name)
        for i, op in enumerate(plan.ops):
            fn, args, name = op[0], op[1], op[2]
            ck = self.rec.by_op.get(id(op))
            if ck is not None and ck.ops[0] is op:
                self._before(ck)
            gctx = self.glue.before(op, i) if (self.glue is not None and ck is None and self.glue.owns(name)) else None
            if fn is None:
                if args is not None:
                    args()
            else:
                _lib.check(fn(*args, st), name)
            if gctx is not None:
                torch.cuda.synchronize()
                self.glue.after(op, gctx)
            if ck is not None and ck.ops[-1] is op:
                torch.cuda.synchronize()
                self._after(ck)
                self.checked += len(ck.ops)
                self.launches[ck.label()] += len(ck.ops)
                if ck.kind == 'wgrad':
                    modes.add(ck.mode)
        torch.cuda.synchronize()
        for mode in modes:
            self._finish_wgrad(mode)

    def _record(self, ck, what, r):
        self.results[ck.label()].append(r)
        if not r <= 1.0:
            self.failures.append('%r: %s bound ratio %.3g' % (ck, what, r))

    def _control(self, name, r):
        if self.controls is not None and name not in self.controls:
            self.controls[name] = r

    # ---- forward
    def _before(self, ck):
        if ck.kind == 'wgrad':
            return self._wgrad_ref(ck)
        i = ck.info
        snap = {}
        for key in ('out', 'tgt'):
            if i.get(key) is not None:
                snap[key] = i[key].buf.clone()
        if i.get('outf') is not None:
            snap['outf'] = i['outf'].clone()
        snap['ref'] = self._fwd_ref(ck) if ck.kind == 'fwd' else self._dgrad_ref(ck)
        self.snap = snap

    def _fwd_ref(self, ck):
        L, i, d = ck.layer, ck.info, ck.descs()[0]
        N = d.N
        x = _concat(i['srcs'], N)
        w = _weights(L)
        y = _conv(L, x, w)
        S = _conv(L, x.abs(), w.abs())
        b = _bias(L)
        y, S = y + b, S + b.abs()
        if i['addf'] is not None:
            a = i['addf'][:N].double()
            y, S = y + a, S + a.abs()
        y = _act(L, y)
        if i['post_add'] is not None:
            p = _real(i['post_add'], N)
            y, S = y + p, S + p.abs()
        gamma = U * max(_conv_terms(q) for q in ck.descs())
        return dict(x=x, w=w, y=y, S=S, gamma=gamma, N=N)

    def _after(self, ck):
        if ck.kind == 'wgrad':
            return
        if ck.kind == 'fwd':
            self._fwd_compare(ck)
        else:
            self._dgrad_compare(ck)
        self.snap = None

    def _fwd_compare(self, ck):
        L, i, s = ck.layer, ck.info, self.snap
        r, d = s['ref'], ck.descs()[0]
        y, S, gamma, N = r['y'], r['S'], r['gamma'], r['N']
        delta = DELTA_ELU if L.act == ACT_ELU else 0.0
        out, outf = i['out'], i['outf']
        if i['mask_mode'] == 1:
            got = outf[:N, ..., 0]
            ref = torch.sigmoid((y[..., 0] - y[..., 1]) / 10.0)
            self._record(ck, 'mask', ratio(got, ref, (S[..., 0] + S[..., 1]) / 40.0, 0.0, gamma, DELTA_MASK))
            self._stray(ck, outf, s['outf'], N, 0, 1, [])
            if out is not None:       # mode 1 stores no bf16 output
                self._stray(ck, out.buf, s['out'], N, 0, 0, [])
            return
        if out is not None:
            got = _real(out, N)
            rr = ratio(got, y, S, E_BF16, gamma * (1 + 2 ** -7), delta * (1 + 2 ** -7))
            self._record(ck, 'bf16 output', rr)
            c0, c1 = d.out_coff, d.out_coff + d.out_ch
            pads = [out.c_off + p for p, m in enumerate(out.chanmap) if m < 0 and c0 <= out.c_off + p < c1]
            self._stray(ck, out.buf, s['out'], N, c0, c1, pads)
            if self.controls is not None:
                self._controls_output(ck, got, rr)
        if outf is not None:
            got = outf[:N, ..., :d.outf_ch]
            self._record(ck, 'fp32 output', ratio(got, y[..., :d.outf_ch], S[..., :d.outf_ch], 0.0, gamma, delta))
            self._stray(ck, outf, s['outf'], N, d.outf_coff, d.outf_coff + d.outf_ch, [])

    def _stray(self, ck, now, old, rows, c0, c1, pads):
        msg = stray(now, old, rows, c0, c1, pads)
        if msg:
            self.failures.append('%r: stray write: %s' % (ck, msg))

    # ---- data gradient
    def _dgrad_ref(self, ck):
        L, i, d = ck.layer, ck.info, ck.descs()[0]
        nb = d.N
        srcs = i['srcs']
        G = _real(i['G'], nb)
        w = _weights(L)
        cin = sum(s.C for s in srcs)
        H, W = srcs[0].H, srcs[0].W
        x = torch.zeros(nb, H, W, cin, dtype=torch.float64, device=G.device, requires_grad=True)
        ref, = torch.autograd.grad(_conv(L, x, w), x, G)
        S, = torch.autograd.grad(_conv(L, x, w.abs()), x, G.abs())
        pre = _real(i['tgt'], nb) if d.add_pre else 0.0
        gamma = U * max(_conv_terms(q) for q in ck.descs())
        return dict(G=G, w=w, ref=ref + pre, S=S + (pre.abs() if d.add_pre else 0.0), gamma=gamma, nb=nb, x=x, pre=pre,
                    add_pre=bool(d.add_pre))

    def _dgrad_compare(self, ck):
        i, s = ck.info, self.snap
        r, d = s['ref'], ck.descs()[0]
        tgt, nb = i['tgt'], r['nb']
        got = _real(tgt, nb)
        rr = ratio(got, r['ref'], r['S'], E_BF16, r['gamma'] * (1 + 2 ** -7), 0.0)
        self._record(ck, 'data gradient', rr)
        c0, c1 = d.out_coff, d.out_coff + d.out_ch
        pads = [tgt.c_off + p for p, m in enumerate(tgt.chanmap) if m < 0 and c0 <= tgt.c_off + p < c1]
        self._stray(ck, tgt.buf, s['tgt'], nb, c0, c1, pads)
        if self.controls is not None:
            self._controls_dgrad(ck, got, rr)

    # ---- weight gradient
    def _wgrad_ref(self, ck):
        L, i, w = ck.layer, ck.info, ck.descs()[0]
        key = (id(L), ck.mode, ck.call, w.tma if not L.transposed else -1)
        terms = _wgrad_terms(w)
        acc = self.wgrad.setdefault((id(L), ck.mode), dict(layer=L, mode=ck.mode, terms=0, checks=[]))
        acc['terms'] = max(acc['terms'], terms)
        acc['checks'].append(ck)
        if key in self.wgrad_seen:          # a second launch of the same call (Cout > 128, transposed parities): same operands
            return
        self.wgrad_seen.add(key)
        nb = w.N
        x = _concat(i['srcs'], nb)
        G = _real(i['G'], nb)
        k = L.k
        shape = (k, k, L.cout, L.cin) if L.transposed else (k, k, L.cin, L.cout)
        wv = torch.zeros(shape, dtype=torch.float64, device=G.device, requires_grad=True)
        dw, = torch.autograd.grad(_conv(L, x, wv), wv, G)
        Sw, = torch.autograd.grad(_conv(L, x.abs(), wv), wv, G.abs())
        db, Sb = G.sum((0, 1, 2)), G.abs().sum((0, 1, 2))
        for name, v in (('dw', dw), ('Sw', Sw), ('db', db), ('Sb', Sb)):
            acc[name] = acc[name] + v if name in acc else v
        acc['npix'] = acc.get('npix', 0) + G.shape[0] * G.shape[1] * G.shape[2]

    def _finish_wgrad(self, mode):
        for key in [k for k in self.wgrad if k[1] == mode]:
            self._wgrad_compare(self.wgrad.pop(key))
        self.wgrad_seen = {k for k in self.wgrad_seen if k[1] != mode}

    def _wgrad_compare(self, acc):
        L, mode, ck = acc['layer'], acc['mode'], acc['checks'][0]
        st = L.store
        nsplit = max([L.wg_splits.get(mode, 0)] + [v for (m, _), v in L.wg_splits_hi.items() if m == mode] +
                     [pk.wg_splits.get(mode, 0) for pk in (L.tr_packs or ())])
        gw = U * (acc['terms'] + nsplit + 4)
        nblk = L.col_blocks[mode]
        gb = U * (-(-acc['npix'] * (4 if L.transposed else 1) // nblk) + nblk + 4)
        dw, Sw, db, Sb = acc['dw'], acc['Sw'], acc['db'], acc['Sb']
        got_w, got_b = st.view(L.wkey, 'grad'), st.view(L.bkey, 'grad')
        if not L.bn:
            rw = ratio(got_w, dw, Sw, 0.0, gw, 0.0)
            rb = ratio(got_b, db, Sb, 0.0, gb, 0.0)
        else:
            wm, bm = st.view(L.wkey).double(), st.view(L.bkey).double()
            g = st.view(L.name + '/gamma').double() * BN_RSQRT
            rw = ratio(got_w, dw * g, Sw * g.abs(), 2.0 ** -22, gw, 0.0)
            rb = max(ratio(got_b, db * g, Sb * g.abs(), 2.0 ** -22, gb, 0.0), ratio(L.db_eff[:L.cout], db, Sb, 0.0, gb, 0.0),
                     ratio(st.view(L.name + '/beta', 'grad'), db, Sb, 0.0, gb, 0.0))
            rows = dw.numel() // L.cout
            dgam = BN_RSQRT * ((dw * wm).reshape(rows, L.cout).sum(0) + db * bm)
            prop = BN_RSQRT * (gw * (Sw * wm.abs()).reshape(rows, L.cout).sum(0) + gb * Sb * bm.abs())
            mag = BN_RSQRT * ((dw * wm).abs().reshape(rows, L.cout).sum(0) + (db * bm).abs())
            got_g = st.view(L.name + '/gamma', 'grad').double()
            rg = float(((got_g - dgam).abs() / (prop + U * (rows // 32 + 32 + 4) * mag + DELTA_FLOOR)).max())
            rb = max(rb, rg if torch.isfinite(got_g).all() else float('inf'))
        for c in acc['checks']:
            self.results[c.label()].append(rw)
        self.results['bias_grad'].append(rb)
        if not rw <= 1.0:
            self.failures.append('%r: weight gradient of %s (mode %s) bound ratio %.3g' % (ck, L.name, mode, rw))
        if not rb <= 1.0:
            self.failures.append('%r: bias / BN gradients of %s (mode %s) bound ratio %.3g' % (ck, L.name, mode, rb))
        if self.controls is not None:
            # the reference without one tap (its bound kept): the stored gradient of that tap must be rejected
            tap = (L.k // 2, L.k // 2)
            ref = dw * (g if L.bn else 1.0)
            S = Sw * (g.abs() if L.bn else 1.0)
            bad = ref.clone()
            bad[tap] = 0
            self._control('wgrad.%s' % ck.label().split('.', 1)[1], ratio(got_w, bad, S, 2.0 ** -22 if L.bn else 0.0, gw, 0.0))

    # ---- negative controls: act on the reference and the copied result only
    def _controls_output(self, ck, got, rr):
        L, r, d = ck.layer, self.snap['ref'], ck.descs()[0]
        if L.transposed or ck.info['mask_mode'] or rr > 1.0:
            return

        def bound_ratio(g, y):    # g against reference y, within the bound of the intact reference
            return ratio(g, y, r['S'], E_BF16, r['gamma'] * (1 + 2 ** -7), DELTA_ELU if L.act == ACT_ELU else 0.0)

        def with_weights(w):
            y = _act(L, _conv(L, r['x'], w) + _bias(L) + (ck.info['addf'][:r['N']].double() if ck.info['addf'] is not None else 0))
            return y + _real(ck.info['post_add'], r['N']) if ck.info['post_add'] is not None else y
        kind = 'fwd.%s' % ('halo' if d.halo else 'gather')
        if kind not in self.controls:
            w = r['w'].clone()
            w[L.k // 2, L.k // 2] = 0          # centre tap dropped; the bound of the intact reference is kept
            self._control(kind, bound_ratio(got, with_weights(w)))
        y = r['y']
        if 'tile' not in self.controls:
            # one 16 x 8 tile of one channel scaled by 1 + 2^-5, at the largest output
            n, h, x, c = [int(v) for v in torch.unravel_index(y.abs().argmax(), y.shape)]
            h0, x0 = h // 16 * 16, x // 8 * 8
            bad = got.clone()
            bad[n, h0:h0 + 16, x0:x0 + 8, c] *= 1 + 2 ** -5
            self._control('tile', bound_ratio(bad, y))
        if d.OW % 8 and 'tile.partial' not in self.controls:
            # the last 16 x 8 tile (partial in x) of one channel scaled by 1 + 2^-5, at the sample and channel where it is largest
            h0, x0 = (d.OH - 1) // 16 * 16, (d.OW - 1) // 8 * 8
            n, c = [int(v) for v in torch.unravel_index(y[:, h0:, x0:].abs().amax((1, 2)).argmax(), (y.shape[0], y.shape[3]))]
            bad = got.clone()
            bad[n, h0:, x0:, c] *= 1 + 2 ** -5
            self._control('tile.partial', bound_ratio(bad, y))
        name = 'thin%d.cin%d' % (d.thin, L.cin)
        if d.thin and L.cin < d.thin and name not in self.controls:
            # the last real input channel dropped (the compact format reads cin real channels and thin - cin zero padding channels)
            w = r['w'].clone()
            w[:, :, L.cin - 1] = 0
            self._control(name, bound_ratio(got, with_weights(w)))

    def _controls_dgrad(self, ck, got, rr):
        L, r, d = ck.layer, self.snap['ref'], ck.descs()[0]
        if d.nsub != 4 or not r['add_pre'] or rr > 1.0 or 'dgrad.parity_group' in self.controls:
            return
        w = r['w'].clone()
        w[L.k // 2, L.k // 2] = 0
        ref, = torch.autograd.grad(_conv(L, r['x'], w), r['x'], r['G'])
        self._control('dgrad.parity_group', ratio(got, ref + r['pre'], r['S'], E_BF16, r['gamma'] * (1 + 2 ** -7), 0.0))

    # ---- summary
    def summary(self):
        """{label: dict(count=launches checked (bias_grad: layer gradients), worst=worst bound ratio)}."""
        return {lab: dict(count=self.launches.get(lab, len(rs)), worst=max(rs)) for lab, rs in sorted(self.results.items())}


def count_persist(rec, plans):
    """label -> (launches, descriptor-side persistent-kernel candidates) over the checks whose ops are in `plans`."""
    ids = {id(op) for p in plans for op in p.ops}
    c = collections.defaultdict(lambda: [0, 0])
    for ck in rec.checks:
        if id(ck.ops[0]) in ids:
            for op in ck.ops:
                d = op[1][0]._obj
                c[ck.label()][0] += 1
                if ck.kind != 'wgrad' and persist_candidate(d):
                    c[ck.label()][1] += 1
    return c


def check_bn_fold(layers):
    """w_eff / b_eff of every BN layer (cis_bn_fold) against the fp64 fold of the master weights -> worst ratio."""
    worst = 0.0
    for L in layers:
        if not L.bn:
            continue
        st = L.store
        g = st.view(L.name + '/gamma').double() * BN_RSQRT
        w = st.view(L.wkey).double() * g
        b = st.view(L.bkey).double() * g
        beta = st.view(L.name + '/beta').double()
        worst = max(worst, ratio(L.w_eff.view(w.shape), w, w.abs(), 2.0 ** -22, 0.0, 0.0),
                    ratio(L.b_eff[:L.cout], b + beta, b.abs() + beta.abs(), 0.0, 2.0 ** -22, 0.0))
    return worst
