"""Static launch-list executor for the hot path: bf16 NHWC activations in HBM, every op a call into libcis_b200.so.

Networks are described once (shapes are static), which produces three launch lists -- forward, backward for the recover
step and backward for the generator step -- that are then replayed (optionally inside a CUDA graph) every iteration.
PyTorch only owns device memory and streams here; there is no autograd and no torch compute on the hot path.
"""
import contextlib
import ctypes as C
import dataclasses
import os

import numpy as np
import torch

from . import _lib
from ._lib import CisConv, CisWgrad, CisSrc, ACT_NONE, ACT_ELU, ACT_LEAKY
from .checkpoint.tf_names import ema_name


def ru(x, m):
    return (x + m - 1) // m * m


def same_pad(n_in, k, s=1, d=1):
    """TF 'SAME' padding split (SURVEY App. A.2)."""
    out = -(-n_in // s)
    total = max((out - 1) * s + (k - 1) * d + 1 - n_in, 0)
    return total // 2, total - total // 2


SIDE_STREAM = True
_SIDE = {}
MULTI_PARAM_OPS = os.environ.get('CIS_MULTI_PARAM', '1') == '1'   # per-layer pack / un-pack / BN launches batched into multi-job launches
DACT_COLSUM = os.environ.get('CIS_DACT_COLSUM', '1') == '1'       # activation derivative and bias-gradient partials of a layer in one launch
PLAN_MODEL = int(os.environ.get('CIS_PLAN_MODEL', '4'))           # MT choice of setup_halo: 1 wave model, 2 busiest-SM model, 3 smallest stack, 4 hybrid (default)
COLSUM_PIX = int(os.environ.get('CIS_COLSUM_PIX', '4'))            # pixels per thread of the column-sum passes (fewer = more blocks, <= 592)


def _side_stream(device, key=0):
    """Side lane of a plan replay.  `key` gives concurrently replayed plans (the pipelined PWC-Net branch) their own lane so the two
    branches do not serialise on one helper stream."""
    k = (str(device), key)
    if k not in _SIDE:
        _SIDE[k] = torch.cuda.Stream(device=device)
    return _SIDE[k]


class Plan(object):
    """An ordered list of C-ABI launches (and a few torch memsets) replayable on any stream."""

    def __init__(self, name=''):
        self.name = name
        self.ops = []
        self.keep = []  # ctypes structs / tensors that must outlive the plan

    def add(self, fname, *args, flops=0.0, lane=0):
        fn = getattr(_lib.load(), fname)
        self.ops.append((fn, args, fname, flops, lane))

    def add_py(self, fn, label='py'):
        self.ops.append((None, fn, label, 0.0, 0))

    def zero(self, t):
        self.keep.append(t)
        self.add('cis_zero', t.data_ptr(), t.numel() * t.element_size())

    def join(self):
        """Main lane waits for everything issued on the side lane so far."""
        self.ops.append((None, None, 'join', 0.0, 0))

    def run(self, stream=None, lane_key=0):
        """Lane 0 = the current stream; lane 1 = a side stream forked/joined with events (weight-gradient GEMMs run there,
        concurrently with the data-gradient chain).  Works eagerly and under CUDA-graph capture."""
        if stream is not None or not SIDE_STREAM or not any(op[4] for op in self.ops):
            st = stream if stream is not None else torch.cuda.current_stream().cuda_stream
            for fn, args, name, _, _ in self.ops:
                if fn is None:
                    if args is not None:
                        args()
                else:
                    rc = fn(*args, st)
                    if rc != 0:
                        _lib.check(rc, name)
            return
        main = torch.cuda.current_stream()
        side = _side_stream(main.device, lane_key)
        st0, st1 = main.cuda_stream, side.cuda_stream
        main_ahead, side_used = True, False
        for fn, args, name, _, lane in self.ops:
            if fn is None:
                if name == 'join':
                    if side_used:
                        ev = torch.cuda.Event()
                        ev.record(side)
                        main.wait_event(ev)
                        side_used = False
                elif args is not None:
                    args()
                    main_ahead = True
                continue
            if lane == 1:
                if main_ahead:
                    ev = torch.cuda.Event()
                    ev.record(main)
                    side.wait_event(ev)
                    main_ahead = False
                rc = fn(*args, st1)
                side_used = True
            else:
                rc = fn(*args, st0)
                main_ahead = True
            if rc != 0:
                _lib.check(rc, name)
        if side_used:
            ev = torch.cuda.Event()
            ev.record(side)
            main.wait_event(ev)

    def batch_param_ops(self, device):
        """A plan made only of the five parameter-space ops (BN fold, weight packs, gradient un-pack, BN chain rule), one launch per
        layer each -> one multi-job launch per kind (cis_param_multi), in dependency order: fold -> packs, un-pack -> chain rule."""
        from ._lib import CisParamJob, JOB_PACK, JOB_PACK_TILED, JOB_UNPACK, JOB_BN_FOLD, JOB_BN_CHAIN
        if not MULTI_PARAM_OPS or not self.ops:
            return self
        jobs = {k: [] for k in range(5)}
        for fn, a, name, _, _ in self.ops:
            j = CisParamJob()
            if name == 'cis_pack_weights':
                w, kmap, K_pad, rows, cout, sn, nmap, wp = a
                j.kind, blocks = JOB_PACK, -(-(rows * K_pad) // 256)
                ptrs, ints = [w, kmap, nmap, wp], [K_pad, rows, cout, sn]
            elif name == 'cis_pack_weights_tiled':
                w, kmap, cin8, ntaps, n_tiles, BN, cout, sn, nmap, out, thin = a
                j.kind, blocks = JOB_PACK_TILED, -(-(n_tiles * (-(-cin8 // 64)) * ntaps * BN * 64) // 256)
                if sn == 1:               # forward orientation: one block per BN x 64 tile (transposed through shared memory)
                    blocks = n_tiles * (-(-cin8 // 64)) * ntaps
                # the compact thin-input tiles are smaller: the kernel walks them over the same blocks
                ptrs, ints = [w, kmap, nmap, out], [cin8, ntaps, n_tiles, BN, cout, sn, thin]
            elif name == 'cis_unpack_wgrad':
                dwp, kmap, K_pad, cout, nsplit, dw, colpart, nblocks, nch, db, layout = a
                j.kind, blocks = JOB_UNPACK, -(-(cout * K_pad + nch) // 256)
                ptrs, ints = [dwp, kmap, dw, colpart, db], [K_pad, cout, nsplit, nblocks, nch, layout]
            elif name == 'cis_bn_fold':
                w, bias, gamma, beta, nw, cout, w_eff, b_eff = a
                j.kind, blocks, j.n = JOB_BN_FOLD, -(-max(nw, cout) // 256), nw
                ptrs, ints = [w, bias, gamma, beta, w_eff, b_eff], [cout]
            elif name == 'cis_bn_chain':
                w, bias, gamma, dwe, dbe, nw, cout, dbias, dgamma, dbeta = a
                j.kind, blocks, j.n = JOB_BN_CHAIN, -(-cout // 8), nw          # one block per 8 output channels (csrc: kBnChainCo)
                ptrs, ints = [w, bias, gamma, dwe, dbe, dbias, dgamma, dbeta], [cout]
            else:
                return self          # something else in the plan: leave it as it is
            for q, v in enumerate(ptrs):
                j.p[q] = v
            for q, v in enumerate(ints):
                j.i[q] = v
            jobs[j.kind].append((j, blocks))
        out = Plan(self.name + '.multi')
        out.keep = self.keep
        for kind in (JOB_BN_FOLD, JOB_PACK_TILED, JOB_PACK, JOB_UNPACK, JOB_BN_CHAIN):
            if not jobs[kind]:
                continue
            arr = (CisParamJob * len(jobs[kind]))()
            first = 0
            for q, (j, blocks) in enumerate(jobs[kind]):
                j.i[7] = first
                arr[q] = j
                first += blocks
            tab = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(device)
            out.keep.append(tab)
            out.add('cis_param_multi', tab.data_ptr(), len(jobs[kind]), first)
        return out

    def count(self):
        """Kernel launches of one replay (a two-launch split-K conv counts twice)."""
        n = 0
        for fn, args, name, _, _ in self.ops:
            if fn is None or name == 'cis_zero':      # a memset node, not a kernel
                continue
            n += 1
            if name == 'cis_conv_igemm':
                d = args[0]._obj
                if d.splits > 1 and not d.sk_cluster:
                    n += 1
        return n

    def extend(self, other):
        self.ops += other.ops
        self.keep += other.keep


class Act(object):
    """A bf16 NHWC activation: a channel slice [c_off, c_off+C8) of a buffer [N,H,W,pitch]."""

    def __init__(self, N, H, W, C, device, buf=None, c_off=0, chanmap=None, n_mod=0, dep=frozenset(), name=''):
        if chanmap is not None and not C:
            C = max(chanmap) + 1
        self.N, self.H, self.W, self.C = N, H, W, C
        self.C8 = ru(C, 8) if chanmap is None else len(chanmap)
        if buf is None:
            buf = torch.zeros(N, H, W, self.C8, dtype=torch.bfloat16, device=device)
        self.buf = buf
        self.pitch = buf.shape[-1]
        self.c_off = c_off
        self.chanmap = list(chanmap) if chanmap is not None else list(range(C)) + [-1] * (self.C8 - C)
        self.n_mod = n_mod
        self.dep = frozenset(dep)
        self.name = name
        self.grad = None
        self.grad_written = {}   # mode -> bool
        self.device = device
        self.gen_rows = None     # batch rows processed by the generator-step backward (2B of 3B)
        self.grad_buf = None     # set: the gradient is the same channel slice of this buffer (views of one zeroed, accumulated buffer)
        self._owner = None       # alias(): the Act whose gradient this view shares

    @property
    def ptr(self):
        return self.buf.data_ptr()

    def src(self):
        return CisSrc(self.ptr, self.pitch, self.c_off, self.C8 // 8, self.n_mod)

    def rows(self, mode):
        return self.gen_rows if (mode == 'G' and self.gen_rows) else self.N

    def alias(self, n_mod):
        """Same storage seen as a batch-broadcast source (features shared by the three recover_net calls)."""
        a = Act(self.N, self.H, self.W, self.C, self.device, buf=self.buf, c_off=self.c_off, chanmap=self.chanmap, n_mod=n_mod,
                dep=self.dep, name=self.name + '.shared')
        a._owner = self
        a.grad_written = self.grad_written
        return a

    def get_grad(self):
        if self._owner is not None:
            return self._owner.get_grad()
        if self.grad is None:
            self.grad = Act(self.N, self.H, self.W, self.C, self.device, buf=self.grad_buf, c_off=self.c_off if self.grad_buf is not None else 0,
                            chanmap=self.chanmap, name=self.name + '.grad')
        return self.grad

    def float(self):
        """Debug/test helper: real channels as fp32 [N,H,W,C] (a torch op, not on the hot path)."""
        idx = [i for i, m in enumerate(self.chanmap) if m >= 0]
        return self.buf[..., self.c_off:self.c_off + self.C8].float()[..., idx]


def _fill_taps(d, taps):
    d.ntaps = len(taps)
    for i, (a, b) in enumerate(taps):
        d.dh[i] = a
        d.dw[i] = b


def _fill_srcs(d, srcs):
    d.nsrc = len(srcs)
    for i, s in enumerate(srcs):
        d.src[i] = s.src()


def conv_desc(N, H, W, OH, OW, stride, taps, srcs, pk, out, out_ch=None, bias=None, act=ACT_NONE, alpha=0.0, grid=None, add_pre=False,
              outf=None, outf_ch=0):
    """A gather-kernel CisConv (setup_halo / setup_halo_s2 may move it to the halo kernel): the N x H x W concat of `srcs` (CisSrc)
    through `taps` at `stride` -> OH x OW, with the row pack of Pack `pk`, bias and activation, into the Act `out` (out_ch channels,
    default its padded width; add_pre: added to what `out` holds) and the fp32 tensor `outf`.  grid = (DH, DW, step, oa, ob): output
    pixel (oh, ow) is pixel (step * oh + oa, step * ow + ob) of a DH x DW map (an output-parity launch); default the OH x OW map."""
    d = CisConv()
    d.N, d.H, d.W, d.OH, d.OW, d.sh, d.sw = N, H, W, OH, OW, stride, stride
    _fill_taps(d, taps)
    d.nsrc = len(srcs)
    for i, s in enumerate(srcs):
        d.src[i] = s
    d.wpack, d.K_pad, d.BN, d.n_tiles = pk.w.data_ptr(), pk.K_pad, pk.BN, pk.n_tiles
    d.bias, d.act, d.alpha = bias, act, alpha
    d.DH, d.DW, step, d.oa, d.ob = grid or (OH, OW, 1, 0, 0)
    d.osh = d.osw = step
    if out is not None:
        d.out, d.out_pitch, d.out_coff, d.out_ch = out.ptr, out.pitch, out.c_off, out.C8 if out_ch is None else out_ch
        if add_pre:
            d.add_pre, d.add_pre_pitch, d.add_pre_coff = out.ptr, out.pitch, out.c_off
    if outf is not None:
        d.outf, d.outf_pitch, d.outf_coff, d.outf_ch = outf.data_ptr(), outf.shape[-1], 0, outf_ch or outf.shape[-1]
    return d


def pick_bn(cout, cap=None):
    """(BN, n_tiles) of the GEMM N dimension.  `cap` (32 / 64) forces narrower n-tiles: more, smaller CTAs for layers whose pixel
    count yields only a handful of 128-row tiles (experiment CIS_SMALL_BN, DESIGN.md section 6 E2)."""
    if cout <= 16:
        return 16, 1
    if cout <= 32:
        return 32, 1
    if cap in (32, 64) and cout > cap:
        return cap, -(-cout // cap)
    if cout <= 64:
        return 64, 1
    return 128, -(-cout // 128)


def small_bn_cap(level):
    """CIS_SMALL_BN="cap:level" (default unset = off): PWC-Net layers of pyramid level >= `level` (12x20 and coarser for level 5)
    use n-tiles of `cap` columns.  Returns the cap for this level or None."""
    spec = os.environ.get('CIS_SMALL_BN', '')
    if not spec:
        return None
    cap, _, lvl = spec.partition(':')
    return int(cap) if level >= int(lvl or 5) else None



NUM_SMS = 132        # H100 SXM
# fp32 accumulator columns (MT stacked tiles x BN) one MMA warpgroup of the halo kernel keeps in its registers
MAX_ACC_COLS = 128
HALO_ENABLED = True
WGRAD_TMA = True
MATERIALIZE_MISALIGNED_CONCAT = True


WGRAD_CTAS_PER_SM = int(os.environ.get('CIS_WGRAD_CTAS_PER_SM', '2'))   # split-K target: CTAs per SM of one weight-gradient launch
WGRAD_MAX_SLICE_MB = float(os.environ.get('CIS_WGRAD_MAX_SLICE_MB', '16'))  # 0 = no cap on splits x Cout x K_pad x 4 bytes per layer
WGRAD_HALO_MIN_CH = int(os.environ.get('CIS_WGRAD_HALO_MIN_CH', '16'))   # thinner inputs: the per-tap 64-channel padding costs more than the gather path
WGRAD_HALO = os.environ.get('CIS_WGRAD_HALO', '1') == '1'   # halo-resident swapped wgrad kernel (CisWgrad.tma = 2) where it fits


def wgrad_halo_fits(taps, cout, stride):
    """Eligibility of the halo-resident wgrad kernel (mirrors launch_wgrad_halo in csrc/conv_igemm.cu): stride 1, taps listed in
    increasing row-major order, (taps/2) x min(Cout16, 64) accumulator columns <= 512 (every CTA along grid.z re-reads the halo:
    larger tap sets are cheaper on the TMA kernel), >= 2 pipeline stages in shared memory.  The tiling is wgrad_halo_tiling's."""
    if stride != 1 or not taps:
        return False
    hoy, hox = min(a for a, _ in taps), min(b for _, b in taps)
    keys = [(a - hoy) * 1024 + (b - hox) for a, b in taps]
    if any(k1 <= k0 for k0, k1 in zip(keys, keys[1:])):
        return False
    wh, hh = 8 + max(b for _, b in taps) - hox, 8 + max(a for a, _ in taps) - hoy
    nh = 64 if cout > 64 else ru(cout, 16)
    if ((len(taps) + 1) // 2) * nh > 512 or wh > 256 or hh > 256:
        return False
    # a stage holds the halo and one 8x8-pixel gradient tile per MMA warpgroup when two warpgroups take the two halves of Cout
    stage = ru(wh * hh * 128, 1024) + 8192 * (2 if WGRAD_HALO_NWG >= 2 and cout > 64 else 1)
    return (200 * 1024) // stage >= 2


# halo wgrad tiling (CisWgrad.nh / nwg).  CIS_WGRAD_HALO_NWG: 1 = N = 64 and one MMA warpgroup of two tap pairs per CTA, split count
# from the input-chunk x Cout-half tiles only (the earlier plan, for A/B runs) | 2 (default) = wgrad_halo_tiling
WGRAD_HALO_NWG = int(os.environ.get('CIS_WGRAD_HALO_NWG', '2'))


def wgrad_splits(nkb, ntile, cout, K_pad):
    """Split-K factor of a weight-gradient launch of nkb reduction blocks and ntile column tiles (grid.x x grid.z)."""
    splits = max(1, min(nkb // 8 if nkb >= 8 else 1, max(1, (WGRAD_CTAS_PER_SM * NUM_SMS) // ntile)))
    if WGRAD_MAX_SLICE_MB > 0:      # the private slices are written once and read once more by the un-pack job: bound their volume
        splits = max(1, min(splits, int(WGRAD_MAX_SLICE_MB * 1e6 / (cout * K_pad * 4.0))))
    return -(-nkb // (-(-nkb // splits)))        # every split owns >= 1 reduction block (its slice is written, not accumulated)


def wgrad_halo_tiling(ntaps, cout):
    """(nh, nwg, grid_z) of a tma = 2 launch (mirrors launch_wgrad_halo_t).  nh = min(64, Cout rounded to 16) is the MMA N, so no MMA
    multiplies zero channels beyond the 16-channel granule; one MMA warpgroup holds 128 // nh tap pairs.  Cout > 64: two warpgroups take
    the two 64-channel halves of Cout over the same pairs (one halo and one gradient stage feed both).  Cout <= 64: a second warpgroup
    when the pairs do not fit one, splitting the CTA's pairs between the two.  grid_z counts the CTAs of one (input chunk, split)."""
    npairs = (ntaps + 1) // 2
    if WGRAD_HALO_NWG < 2:
        return 64, 1, (2 if cout > 64 else 1) * (-(-npairs // 2))
    nh = 64 if cout > 64 else ru(cout, 16)
    p = MAX_ACC_COLS // nh
    if cout > 64:
        return 64, 2, -(-npairs // p)
    nwg = 2 if npairs > p else 1
    return nh, nwg, -(-npairs // (nwg * p))




# split-K of launches that cover only a few SMs (low-resolution pyramid levels): 0 = off, 2 = on (two launches: private partial slices +
# a parallel finish kernel with a fixed summation order)
SPLITK = int(os.environ.get('CIS_SPLITK', '2'))
SPLITK_CLUSTER = os.environ.get('CIS_SPLITK_CLUSTER', '0') == '1'   # reduce through a thread-block cluster (DSMEM) instead of the finish launch
SPLITK_MAX = int(os.environ.get('CIS_SPLITK_MAX', '16'))
SPLITK_NCTA = int(os.environ.get('CIS_SPLITK_NCTA', '64'))          # only launches with at most this many CTAs are split
SPLITK_MIN_UNITS = int(os.environ.get('CIS_SPLITK_MIN_UNITS', '18'))  # ... and at least this many serial pipeline steps per CTA
# experiment switch (default off = current behaviour): stride-1 layers whose padded input width is <= this many channels and that
# have >= 16 taps (generator conv1 5x5x8, recover flow1 5x5) use the K-dense gather kernel (ceil(taps*cin8/64) pipeline steps)
# instead of the halo kernel (one step and one mostly-zero BN x 128 B weight tile per tap); see DESIGN.md section 6, E1
HALO_SKIP_THIN = int(os.environ.get('CIS_HALO_SKIP_THIN', '0'))
# smallest useful fraction of a launch's 16x8 output tiles for the halo kernel to take a stride-1 layer (below it: the K-dense gather
# kernel).  Low-resolution maps (6x10, 8x14, 4x7) only fill 20-45 % of their tiles, but the gather kernel's cp.async producers cost
# several times more per 64-wide K block than the halo kernel spends on a stage of taps
HALO_MIN_UTIL = float(os.environ.get('CIS_HALO_MIN_UTIL', '0.2'))


# MMA warpgroups per halo-kernel CTA (CisConv.nwg): 2 = both warpgroups consume every weight stage, so the CTA pulls half the weight
# bytes from L2 per output row.  CIS_HALO_NWG: 1 one warpgroup everywhere (A/B runs) | 2 (default) where halo_nwg's rule says it pays |
# 3 every launch that can take two (tests)
HALO_NWG = int(os.environ.get('CIS_HALO_NWG', '2'))
# time of a two-warpgroup CTA relative to two one-warpgroup CTAs of the same rows: 0.78-0.80 measured on the 4x96x160 BN = 128 PWC-Net
# layers (H100 SXM at a 400 W power limit, tools/time_ops.py)
HALO_NWG2_COST = 0.8


def halo_nwg(d, MT, Hp0, Wp0, dil, n_tiles, ntaps, nchunks, ey, ex):
    """CisConv.nwg for a halo launch of MT tiles per warpgroup: 2 when the launch spans more than one wave of CTAs, so that half as
    many CTAs of twice the height take fewer waves-times-cost, the taller tile wastes no more padded rows and the taller halo fits
    shared memory; else 1."""
    if HALO_NWG < 2 or d.BN < 64:
        return 1
    if HALO_NWG == 2 and n_tiles == 1 and dil == 1 and MT * d.BN <= 64 and nchunks * ntaps * d.BN * 128 <= 112 * 1024:
        return 1           # a candidate of the persistent kernel (one warpgroup, whole weight set resident in shared memory)
    tiles_x = -(-Wp0 // 8)
    ty1, ty2 = -(-Hp0 // (16 * MT)), -(-Hp0 // (32 * MT))
    HP = (8 + ex) * (32 * MT + ey)
    nhs = 2 if nchunks > 1 else 1
    if nhs * ru(HP * 128, 1024) + HP * 4 + 2048 + 3 * d.BN * 128 > 227 * 1024 or 2 * MT * 128 * d.BN * 4 + 1024 > 226 * 1024:
        return 1
    util1 = (Hp0 * Wp0) / float(ty1 * 16 * MT * tiles_x * 8)
    util2 = (Hp0 * Wp0) / float(ty2 * 32 * MT * tiles_x * 8)
    if util2 < (HALO_MIN_UTIL if dil == 1 else 0.5):
        return 1
    if HALO_NWG == 3:
        return 2
    if util2 < 0.95 * util1:
        return 1
    # one CTA per SM either way (register-bound): compare whole waves of CTAs, a two-warpgroup CTA costing 2 * HALO_NWG2_COST
    ncta1 = d.N * dil * dil * tiles_x * ty1 * n_tiles
    ncta2 = d.N * dil * dil * tiles_x * ty2 * n_tiles
    return 2 if 2 * HALO_NWG2_COST * (-(-ncta2 // NUM_SMS)) <= -(-ncta1 // NUM_SMS) else 1


def setup_splitk(d, device, keep):
    """Launches whose grid would cover well under the NUM_SMS SMs (low-resolution pyramid levels) split their K loop over grid.z;
    see CisConv.splits.  Scratch and ticket buffers are per launch (launches on different lanes may overlap)."""
    if not SPLITK:
        return
    m_chunks = sum(d.src[i].chunks for i in range(d.nsrc))
    if d.halo:
        Hp0, Wp0 = -(-d.OH // d.dil), -(-d.OW // d.dil)
        mt = d.MT * max(d.nwg, 1)         # 16x8 tiles per CTA
        tiles = (-(-Wp0 // 8)) * (-(-Hp0 // (16 * mt))) * d.dil * d.dil * d.N
        ncta, units, min_units = tiles * d.n_tiles, -(-m_chunks // 8), 1
    else:
        ncta, units, min_units, mt = (-(-(d.N * d.OH * d.OW) // 128)) * d.n_tiles, d.K_pad // 64, 4, 1
    steps = units * (d.ntaps if d.halo else 1)     # serial pipeline steps of one CTA (halo: one per (chunk, tap); generic: one per 64-wide K block)
    if ncta > SPLITK_NCTA or steps < SPLITK_MIN_UNITS:
        return
    splits = min(units // min_units, -(-2 * NUM_SMS // ncta), SPLITK_MAX, 8 if SPLITK_CLUSTER else 1 << 30)
    if splits < 2:
        return
    per = -(-units // splits)
    splits = -(-units // per)
    if splits < 2:
        return
    if SPLITK_CLUSTER and splits <= 8 and mt * 128 * d.BN * 4 + 1024 <= 226 * 1024:
        # the splits of a tile form a thread-block cluster and reduce through distributed shared memory: no scratch, no second launch
        d.splits, d.sk_scratch, d.sk_counters, d.sk_cluster = splits, None, None, 1
        return
    sc = torch.empty(ncta * mt * splits * 128 * d.BN, dtype=torch.float32, device=device)
    keep.append(sc)
    d.splits, d.sk_scratch, d.sk_counters = splits, sc.data_ptr(), None


def setup_halo(d, taps, dil, n_tiles):
    """Switch a stride-1 gather descriptor to the halo-resident kernel when it pays off: taps become offsets relative to the
    halo origin in units of `dil`, MT (stacked 16x8 tiles per CTA) is chosen by a wave/overhead model."""
    if not HALO_ENABLED or d.sh != 1 or d.sw != 1:
        return False
    if any(a % dil or b % dil for a, b in taps):
        return False
    if dil > 1 and (d.OH != d.H or d.OW != d.W):
        return False
    th = [(a // dil, b // dil) for a, b in taps]
    hoy, hox = min(a for a, _ in th), min(b for _, b in th)
    rel = [(a - hoy, b - hox) for a, b in th]
    ey, ex = max(a for a, _ in rel), max(b for _, b in rel)
    Hp0, Wp0 = -(-d.OH // dil), -(-d.OW // dil)
    tiles_x = -(-Wp0 // 8)
    best = None
    ntaps = len(taps)
    m_chunks = sum(d.src[i].chunks for i in range(d.nsrc))
    if HALO_SKIP_THIN and m_chunks * 8 <= HALO_SKIP_THIN and ntaps >= 16:
        return False
    nchunks = -(-m_chunks // 8)
    nhs = 2 if nchunks > 1 else 1
    force = int(os.environ.get('CIS_FORCE_MT128', '0')) if d.BN == 128 else 0
    for MT in (1, 2, 3, 4):
        if MT * d.BN > MAX_ACC_COLS or (force and MT != force):
            continue
        HP = (8 + ex) * (16 * MT + ey)
        fixed = nhs * ru(HP * 128, 1024) + HP * 4 + 1024
        smem = fixed + min(3, ntaps * nchunks) * d.BN * 128 + 1024
        if smem > 227 * 1024:
            continue
        tiles_y = -(-Hp0 // (16 * MT))
        util = (Hp0 * Wp0) / float(tiles_y * 16 * MT * tiles_x * 8)
        if util < (HALO_MIN_UTIL if dil == 1 else 0.5):      # dilated phases: no TMA halo path, d*d times the CTAs -> keep the old rule
            continue
        ncta = d.N * dil * dil * tiles_x * tiles_y * n_tiles
        cps = max(1, min((225 * 1024) // smem, 6))
        # per CTA: tensor time vs operand traffic (weights through the TMA engine ~40 B/clk/SM, halo through LDGSTS ~16 B/clk/SM),
        # plus a fixed prologue/epilogue latency that co-resident CTAs overlap
        t_mma = MT * 2.0 * d.BN * ntaps * nchunks
        t_mem = (d.BN * 128 * ntaps / 40.0 + HP * 128 / 16.0) * nchunks
        t_cta = max(t_mma, t_mem) + (4000.0 + 1500.0 * MT) / cps
        cost = -(-ncta // (NUM_SMS * cps)) * cps * t_cta / min(cps, max(1.0, ncta / float(NUM_SMS)))
        if PLAN_MODEL == 2:
            # busiest SM: its CTAs' throughput-bound parts add up, their fixed latencies overlap cps at a time
            per_sm = -(-ncta // NUM_SMS)
            cost = per_sm * max(t_mma, t_mem) + (4000.0 + 1500.0 * MT) * (-(-per_sm // cps))
        if PLAN_MODEL == 3:
            cost = float(MT)            # smallest feasible stack
        if PLAN_MODEL == 4:
            # from an A/B of models 1-3 over every layer of the step: the smallest feasible stack wins everywhere EXCEPT on
            # big grids of short tiles (MMA loop below the fixed prologue + epilogue of a CTA), where the wave model's choice holds
            n1 = d.N * dil * dil * tiles_x * (-(-Hp0 // 16)) * n_tiles
            if not (2.0 * d.BN * ntaps * nchunks < 6000.0 and n1 > 4 * NUM_SMS):
                cost = float(MT)
        if best is None or cost < best[0] - 1e-9:
            best = (cost, MT, util)
    if best is None:
        return False
    d.halo, d.dil, d.MT, d.hoy, d.hox, d.ey, d.ex = 1, dil, best[1], hoy, hox, ey, ex
    d.nwg = halo_nwg(d, best[1], Hp0, Wp0, dil, n_tiles, ntaps, nchunks, ey, ex)
    d.thin = thin_format(m_chunks, dil)
    _fill_taps(d, [rel[i] for i in thin_tap_order(d.thin, rel)])
    return True


def thin_format(m_chunks, dil):
    """CisConv.thin of an undilated halo launch whose sources total m_chunks 8-channel chunks: 8 or 16 channels take the compact K-dense
    format (a 16-byte-per-pixel halo; one K=16 step per tap pair or per tap instead of one per tap of a mostly-zero 64-channel chunk)."""
    return m_chunks * 8 if dil == 1 and m_chunks in (1, 2) else 0


def thin_tap_order(thin, taps):
    """Order of the taps in a halo launch and in its pre-tiled weights: the compact 8-channel format pairs consecutive taps in one K=16
    step whose second tap must lie at a positive offset from the first, so it lists them in increasing (dy, dx); else as given."""
    return sorted(range(len(taps)), key=lambda i: tuple(taps[i])) if thin == 8 else list(range(len(taps)))


# stride-2 forward convolutions on the halo kernel (4 space-to-depth phase tensor maps, CisConv.nph = 4).  Off by default: every tap
# of the thin 7x7 / 5x5 first layers pays a whole 64-channel chunk there -- the K-dense gather kernel stays the stride-2 path.
S2_HALO = os.environ.get('CIS_S2_HALO', '0') == '1'


def setup_halo_s2(d, taps, n_tiles):
    """Stride-2 forward conv as a halo-kernel launch: input pixel (2*oh + u, 2*ow + v) of tap (u, v) is pixel (oh + u // 2, ow + v // 2)
    of the space-to-depth phase (u % 2, v % 2), so the conv is the sum over the 4 phases of stride-1 convs with the taps of that phase.
    Returns the tap permutation (phase-major) the pre-tiled weights must follow, or None when the launch stays on the gather kernel."""
    if not (HALO_ENABLED and S2_HALO) or d.sh != 2 or d.sw != 2:
        return None
    if any(d.src[i].chunks % 8 for i in range(d.nsrc - 1)):       # TMA halo path only: a 64-channel chunk never straddles sources
        return None
    ph = [((u % 2) * 2 + (v % 2), u // 2, v // 2) for u, v in taps]
    order = sorted(range(len(taps)), key=lambda i: (ph[i][0], i))
    hoy, hox = min(a for _, a, _ in ph), min(b for _, _, b in ph)
    rel = [(ph[i][1] - hoy, ph[i][2] - hox) for i in order]
    ey, ex = max(a for a, _ in rel), max(b for _, b in rel)
    m_chunks = sum(d.src[i].chunks for i in range(d.nsrc))
    nchunks = -(-m_chunks // 8)
    tiles_x = -(-d.OW // 8)
    best = None
    for MT in (1, 2, 3, 4):
        if MT * d.BN > MAX_ACC_COLS:
            continue
        HP = (8 + ex) * (16 * MT + ey)
        smem = 2 * ru(HP * 128, 1024) + HP * 4 + 2048 + 2 * d.BN * 128
        if smem > 227 * 1024:
            continue
        tiles_y = -(-d.OH // (16 * MT))
        util = (d.OH * d.OW) / float(tiles_y * 16 * MT * tiles_x * 8)
        if util < HALO_MIN_UTIL:
            continue
        ncta = d.N * tiles_x * tiles_y * n_tiles
        cps = max(1, min((225 * 1024) // smem, 4))
        t_mma = MT * 2.0 * d.BN * len(taps) * nchunks
        t_mem = (d.BN * 128 * len(taps) / 40.0 + 4 * HP * 128 / 40.0) * nchunks
        t_cta = max(t_mma, t_mem) + (4000.0 + 1500.0 * MT) / cps
        cost = -(-ncta // (NUM_SMS * cps)) * cps * t_cta / min(cps, max(1.0, ncta / float(NUM_SMS)))
        if best is None or cost < best[0] - 1e-9:
            best = (cost, MT)
    if best is None:
        return None
    d.halo, d.dil, d.MT, d.hoy, d.hox, d.ey, d.ex = 1, 1, best[1], hoy, hox, ey, ex
    d.nwg = halo_nwg(d, best[1], d.OH, d.OW, 1, n_tiles, len(taps), nchunks, ey, ex)
    d.sh = d.sw = 1                     # the phases absorb the stride; H x W stay the input size (tensor maps)
    _fill_taps(d, rel)
    d.nph = 4
    bounds = [0]
    for q in range(4):
        bounds.append(bounds[-1] + sum(1 for i in order if ph[i][0] == q))
    for q in range(5):
        d.ph_tap[q] = bounds[q]
    return order


GROUP_PARITY = os.environ.get('CIS_GROUP_PARITY', '1') == '1'   # the 4 output-parity launches of a stride-2 dgrad / transposed conv as one
GROUP_PARITY_MAX_TILES = int(os.environ.get('CIS_GROUP_PARITY_MAX_TILES', '1000000'))   # optional cap on the 16x8 tiles per parity (600: +0.4 % device-resident, within noise end to end)


def merge_parity_launches(descs):
    """Four (or fewer) halo-kernel descriptors that differ only in taps / halo origin / weights / output extent and offset -> ONE grouped
    descriptor (CisConv.nsub), or None when they cannot share a launch."""
    if not GROUP_PARITY or not (2 <= len(descs) <= 4):
        return None
    d0 = descs[0]
    same = ('N', 'H', 'W', 'BN', 'n_tiles', 'nsrc', 'act', 'DH', 'DW', 'osh', 'osw', 'out', 'out_pitch', 'out_coff', 'out_ch', 'outf', 'outf_pitch',
            'outf_coff', 'outf_ch', 'add_pre', 'add_pre_pitch', 'add_pre_coff', 'add_post', 'addf_pre', 'mode', 'bias', 'thin')
    for d in descs:
        if not d.halo or d.dil != 1 or d.splits > 1 or d.nph > 1 or any(getattr(d, f) != getattr(d0, f) for f in same):
            return None
        if any(bytes(d.src[i]) != bytes(d0.src[i]) for i in range(d0.nsrc)):
            return None
    if sum(d.ntaps for d in descs) > _lib.MAX_TAPS:
        return None
    # big grids are better off as separate launches (each becomes a persistent weight-resident launch when it qualifies): grouping
    # pays below ~600 tiles per parity (one launch instead of four latency-bound ones)
    if max(d.N * (-(-d.OH // 16)) * (-(-d.OW // 8)) for d in descs) > GROUP_PARITY_MAX_TILES:
        return None
    g = CisConv.from_buffer_copy(bytes(d0))
    g.MT, g.ey, g.ex = min(d.MT for d in descs), max(d.ey for d in descs), max(d.ex for d in descs)
    g.nwg = min(max(d.nwg, 1) for d in descs)
    g.OH, g.OW = max(d.OH for d in descs), max(d.OW for d in descs)
    t = 0
    for i, d in enumerate(descs):
        for k in range(d.ntaps):
            g.dh[t + k], g.dw[t + k] = d.dh[k], d.dw[k]
        sb = g.sub[i]
        sb.tap0, sb.ntaps, sb.hoy, sb.hox, sb.OH, sb.OW, sb.oa, sb.ob, sb.wpack = t, d.ntaps, d.hoy, d.hox, d.OH, d.OW, d.oa, d.ob, d.wpack
        t += d.ntaps
    m_chunks = sum(g.src[i].chunks for i in range(g.nsrc))
    g.ntaps, g.nsub, g.splits, g.K_pad = t, len(descs), 0, ru(t * m_chunks * 8, 64)
    return g


class ParamStore(object):
    """One flat fp32 parameter buffer (+ grad, Adam m/v) per variable scope; names follow the TF variable layout
    (adversarial_learner.py:211-214 scopes 'MaskNet' / 'FlownetS'; model_pwcnet.py 'pwcnet').  add_shadow() adds `shadow`, the moving
    average of `flat` (cis_ema_update), in the same layout."""

    def __init__(self, device):
        self.device = device
        self.entries = []   # (name, shape, real_numel, offset, padded_numel)
        self.index = {}
        self.size = 0
        self.flat = None
        self.shadow = None

    def declare(self, name, shape, padded=None):
        n = int(np.prod(shape))
        pn = ru(padded or n, 4)
        self.index[name] = len(self.entries)
        self.entries.append((name, tuple(shape), n, self.size, pn))
        self.size += pn

    def finalize(self, trainable):
        self.flat = torch.zeros(self.size, dtype=torch.float32, device=self.device)
        if trainable:
            self.grad = torch.zeros_like(self.flat)
            self.m = torch.zeros_like(self.flat)
            self.v = torch.zeros_like(self.flat)
            seg = [0]
            for _, _, n, off, _ in self.entries:
                seg.append(off + n)
            # segment i = [offset_i, offset_i + n_i): built as explicit (start,end) pairs flattened for the kernel
            self.seg_pairs = [(off, off + n) for _, _, n, off, _ in self.entries]

    def off(self, name):
        return self.entries[self.index[name]][3]

    def ptr(self, name, which='flat'):
        return getattr(self, which).data_ptr() + 4 * self.off(name)

    def view(self, name, which='flat'):
        _, shape, n, off, _ = self.entries[self.index[name]]
        return getattr(self, which)[off:off + n].view(shape)

    def add_shadow(self):
        """Allocate `shadow`, initialised from flat (padding included, so padded entries stay 0)."""
        self.shadow = self.flat.clone()

    def load(self, params):
        """Every variable from params[name]; with a shadow, its moving average from params[ema_name(name)], or from the loaded value
        when params has none."""
        for name, shape, n, off, _ in self.entries:
            if name not in params:
                raise KeyError('missing parameter ' + name)
            self.flat[off:off + n].copy_(self._flat_value(params, name, n))
            if self.shadow is not None:
                avg = ema_name(name)
                self.shadow[off:off + n].copy_(self._flat_value(params, avg, n) if avg in params else self.flat[off:off + n])

    @staticmethod
    def _flat_value(params, name, n):
        t = params[name].detach().to(torch.float32).reshape(-1)
        if t.numel() != n:
            raise ValueError('shape mismatch for %s: %d vs %d' % (name, t.numel(), n))
        return t

    def export(self, which='flat'):
        return {name: getattr(self, which)[off:off + n].view(shape).clone() for name, shape, n, off, _ in self.entries}

    def export_all(self):
        """export() plus, with a shadow, every moving average under its ema_name: what a checkpoint of this store holds."""
        out = self.export()
        if self.shadow is not None:
            out.update((ema_name(k), v) for k, v in self.export('shadow').items())
        return out

    def real_count(self):
        return sum(e[2] for e in self.entries)


def check_ema_decay(decay):
    """ValueError unless decay is 0 (no moving average) or 0 < decay < 1."""
    if not (decay == 0 or 0 < decay < 1):
        raise ValueError('ema_decay must be 0 (off) or in (0, 1), got %r' % (decay,))


@contextlib.contextmanager
def averaged_weights(graph, stores):
    """Inside the block the flat buffer of each of `stores` holds its moving average (shadow), and graph._dirty makes the graph rebuild
    its packed bf16 operands from it on first use.  The packs alone would not do: a conv without batch norm reads its bias from flat
    when it runs.  On exit the live weights are copied back, bit for bit, and the operands marked for a re-pack, so training continues
    from the live weights.  No stores: nothing changes."""
    if not stores:
        yield
        return
    live = [s.flat.clone() for s in stores]
    for s in stores:
        s.flat.copy_(s.shadow)
    graph._dirty = True
    try:
        yield
    finally:
        for s, t in zip(stores, live):
            s.flat.copy_(t)
        graph._dirty = True


@dataclasses.dataclass(eq=False)
class Pack:
    """One packed bf16 weight operand of a conv layer.  a, b: output parity of a parity launch; taps: its (dy, dx) offsets (forward
    operand: the tap indices, in its tiled copy's order); kmap: packed K position -> flat weight offset; w: row pack [rows][K_pad] of
    the gather kernel; nmap: row -> output channel (None = identity); wt: tiled copy of the halo kernel, allocated when the first launch
    goes there, wt_kmap its kmap if the tap order differs, thin its CisConv.thin format; rows_used: None until a launch is placed (rows packed), False while only halo
    launches read the operand; wg_splits / dwp: per-mode split count and fp32 slices of the parity's weight gradient (transposed conv)."""
    a: int = 0
    b: int = 0
    taps: list = dataclasses.field(default_factory=list)
    kmap: torch.Tensor = None
    K_pad: int = 0
    rows: int = 0
    BN: int = 0
    n_tiles: int = 0
    nmap: torch.Tensor = None
    w: torch.Tensor = None
    wt: torch.Tensor = None
    wt_kmap: torch.Tensor = None
    thin: int = 0
    rows_used: bool = None
    wg_splits: dict = dataclasses.field(default_factory=dict)
    dwp: torch.Tensor = None

    def __getitem__(self, field):       # read access by field name, as for the pack dicts this record replaced
        return getattr(self, field)


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _parity_taps(k, s, d, pt, pl, a, b):
    """Taps of a k x k conv (stride s, dilation d, pt / pl rows / columns of padding in front) that connect input pixels of parity
    (a, b) to output pixels: input (s y + a, s x + b) meets output (y + dy, x + dx) through tap r * k + c.  -> (indices, offsets)."""
    rows = [r for r in range(k) if (a + pt - r * d) % s == 0]
    cols = [c for c in range(k) if (b + pl - c * d) % s == 0]
    return [r * k + c for r in rows for c in cols], [((a + pt - r * d) // s, (b + pl - c * d) // s) for r in rows for c in cols]


class ConvLayer(object):
    """One conv layer's static data: parameter views, packed bf16 operands (forward and data-gradient orientation),
    the fp32 packed weight-gradient buffer and the channel maps that tie packed K positions to HWIO indices."""

    def __init__(self, store, name, k, cin, cout, stride=1, dil=1, act=ACT_NONE, alpha=0.2, tag='', bn=False,
                 wname='kernel', bname='bias', transposed=False, bn_cap=None):
        self.store, self.name, self.k, self.cin, self.cout = store, name, k, cin, cout
        self.stride, self.dil, self.act, self.alpha, self.tag, self.bn = stride, dil, act, alpha, tag, bn
        self.transposed = transposed
        self.bn_cap = bn_cap
        self.BN, self.n_tiles = pick_bn(cout, bn_cap)
        self.npad = self.BN * self.n_tiles
        self.wkey, self.bkey = '%s/%s' % (name, wname), '%s/%s' % (name, bname)
        if transposed:
            store.declare(self.wkey, (k, k, cout, cin))
        else:
            store.declare(self.wkey, (k, k, cin, cout))
        store.declare(self.bkey, (cout,), padded=self.npad)
        if bn:
            store.declare('%s/gamma' % name, (cout,))
            store.declare('%s/beta' % name, (cout,))
        self.device = store.device
        # set up by the first launch that needs them
        self.in_chanmap = None          # packed input position -> input channel
        self.fwd_kmap, self.K_pad = None, 0            # forward K layout: packed K position -> flat HWIO offset (setup_fwd)
        self.fwd_pack = None            # Pack of the forward operand (setup_fwd)
        self.tr_packs = None            # transposed conv: the four output-parity Packs of the forward (setup_transposed)
        self.dgrad_packs = None         # data gradient: one Pack per input parity (setup_dgrad)
        self.tr_dgrad = None            # transposed conv: the Pack of the data gradient (setup_transposed_dgrad)
        self.dgrad_used = False         # a data-gradient launch was emitted
        self.w_eff = self.b_eff = self.db_eff = None     # BN: folded weights and bias, gradient of the folded bias
        self.ncalls = 0                 # forward calls with a backward (the siamese PWC-Net feature pyramid runs twice)
        self.colpart, self.col_blocks = None, {}         # bias-gradient partials of every call, their block count per mode
        self.tr_planes = None           # transposed conv: the output gradient split into its four output-parity planes
        self.dcat = None                # gradient of a multi-source input (the virtual concat)
        # weight gradient (setup_wgrad): kernel path and packed K layout; per mode the split count of the fp32 slice buffers
        self.wg_tma = self.wg_halo = False
        self.wg_kmap, self.wg_K_pad = None, 0
        self.dwp, self.wg_splits = None, {}
        self.dwp_hi, self.wg_splits_hi = {}, {}   # Cout > 128: output channels [g0, g0 + 128), g0 >= 128, in launches of their own
        self.wgrad_modes = set()

    # ---- packed operands -------------------------------------------------------------------------------------
    def _kmap(self, taps_idx, chanmap, per_tap_stride, chan_stride):
        """kmap[k=(ti,pos)] = taps_idx[ti]*per_tap_stride + chanmap[pos]*chan_stride (or -1)."""
        m = len(chanmap)
        K = len(taps_idx) * m
        Kp = ru(max(K, (len(taps_idx) - 1) * m + ru(m, 64)), 64)   # halo kernel reads 64-channel chunks per tap
        km = np.full(Kp, -1, dtype=np.int32)
        cm = np.asarray(chanmap, dtype=np.int64)
        for ti, t in enumerate(taps_idx):
            v = np.where(cm >= 0, t * per_tap_stride + cm * chan_stride, -1)
            km[ti * m:(ti + 1) * m] = v
        return torch.from_numpy(km).to(self.device), Kp

    def _rows(self, rows, K_pad):
        return torch.zeros(rows, K_pad, dtype=torch.bfloat16, device=self.device)

    def setup_fwd(self, chanmap):
        """chanmap: packed input position -> original input channel (or -1)."""
        assert max(chanmap) == self.cin - 1, (self.name, max(chanmap), self.cin)
        self.in_chanmap = list(chanmap)
        kk = self.k * self.k
        if self.transposed:
            raise RuntimeError('use setup_transposed')
        self.fwd_kmap, self.K_pad = self._kmap(range(kk), chanmap, self.cin * self.cout, self.cout)
        self.fwd_pack = Pack(taps=list(range(kk)), kmap=self.fwd_kmap, K_pad=self.K_pad, rows=self.npad, BN=self.BN, n_tiles=self.n_tiles,
                             w=self._rows(self.npad, self.K_pad))
        if self.bn:
            self.w_eff = torch.zeros(kk * self.cin * self.cout, dtype=torch.float32, device=self.device)
            self.b_eff = torch.zeros(self.npad, dtype=torch.float32, device=self.device)
            self.db_eff = torch.zeros(self.npad, dtype=torch.float32, device=self.device)

    def _alloc_tiles(self, ntaps, cin8, BN, n_tiles):
        nchunks = -(-cin8 // 64)
        return torch.zeros(n_tiles * nchunks * ntaps * BN * 64, dtype=torch.bfloat16, device=self.device)

    def place(self, d, pk, taps, dil, kch, order=None):
        """Put launch `d` of operand `pk` (kch channels along K) on the halo kernel when setup_halo takes it -- or setup_halo_s2 already
        did and gave the phase-major tap `order` -- reading the operand's pre-swizzled tiled copy, else leave it on the gather kernel."""
        if order is None and not setup_halo(d, taps, dil, pk.n_tiles):
            pk.rows_used = True
            return
        if pk.wt is None:
            pk.wt = self._alloc_tiles(len(taps), kch, pk.BN, pk.n_tiles)
            pk.thin = d.thin
            if order is not None:
                pk.taps = list(order)
                pk.wt_kmap, _ = self._kmap(pk.taps, self.in_chanmap, self.cin * self.cout, self.cout)
            perm = thin_tap_order(d.thin, taps)
            if perm != sorted(perm):         # the compact 8-channel tiles follow the launch's tap order
                n = len(taps)
                pk.wt_kmap = pk.kmap.clone()
                pk.wt_kmap[:n * kch] = pk.kmap[:n * kch].view(n, kch)[perm].reshape(-1)
        assert order is None or pk.taps == list(order), self.name
        assert pk.thin == d.thin, self.name
        d.wpack = pk.wt.data_ptr()
        if pk.rows_used is None:
            pk.rows_used = False

    def w_src_ptr(self):
        return self.w_eff.data_ptr() if self.bn else self.store.ptr(self.wkey)

    def bias_ptr(self):
        return self.b_eff.data_ptr() if self.bn else self.store.ptr(self.bkey)

    def plan_pack(self, plan, dgrad=False):
        """(Re)build the packed bf16 operands from the fp32 master weights."""
        s = self.store
        if self.bn:
            plan.add('cis_bn_fold', s.ptr(self.wkey), s.ptr(self.bkey), s.ptr(self.name + '/gamma'), s.ptr(self.name + '/beta'),
                     self.k * self.k * self.cin * self.cout, self.cout, self.w_eff.data_ptr(), self.b_eff.data_ptr())
        cin8 = len(self.in_chanmap or ())
        # (pack, channels along K, output channels, n stride of the weights): a transposed conv's [kh,kw,Cout,Cin] weights have n stride
        # Cin; its data gradient reads them as the HWIO weights of a stride-2 conv Cout -> Cin
        packs = [(pk, cin8, self.cout, self.cin) for pk in self.tr_packs or ()]
        packs += [(pk, cin8, self.cout, 1) for pk in (self.fwd_pack,) if pk is not None]
        if dgrad:
            packs += [(pk, cin8, cin8, 1) for pk in (self.tr_dgrad,) if pk is not None]
            packs += [(pk, ru(self.cout, 8), cin8, self.cout) for pk in self.dgrad_packs or ()]
        for pk, kch, nch, sn in packs:
            if pk.wt is not None:
                plan.add('cis_pack_weights_tiled', self.w_src_ptr(), (pk.kmap if pk.wt_kmap is None else pk.wt_kmap).data_ptr(), kch,
                         len(pk.taps), pk.n_tiles, pk.BN, nch, sn, _ptr(pk.nmap), pk.wt.data_ptr(), pk.thin)
            if pk.rows_used is not False:
                plan.add('cis_pack_weights', self.w_src_ptr(), pk.kmap.data_ptr(), pk.K_pad, pk.rows, nch, sn, _ptr(pk.nmap), pk.w.data_ptr())

    def plan_finalize(self, bp, mode):
        """Fixed-order sum of the private split-K slices of the packed fp32 weight gradient -> HWIO slot of the flat gradient
        buffer, same for the per-block bias-gradient partials (+ BN chain rule for the generator).  No atomics, nothing to zero."""
        s = self.store
        if self.transposed:
            # four output-parity weight gradients, each into its own taps of the [kh,kw,Cout,Cin] slot (n stride Cin: layout bits 8+); the
            # first also sums the bias partials of the whole output gradient
            for q, pk in enumerate(p for p in self.tr_packs or () if mode in p.wg_splits):
                bp.add('cis_unpack_wgrad', pk.dwp.data_ptr(), pk.kmap.data_ptr(), pk.K_pad, self.cout, pk.wg_splits[mode],
                       s.ptr(self.wkey, 'grad'), self.colpart.data_ptr() if q == 0 else None, self.col_blocks[mode] if q == 0 else 0,
                       self.cout if q == 0 else 0, s.ptr(self.bkey, 'grad') if q == 0 else None, 1 | (self.cin << 8))
            return
        if mode not in self.wg_splits:
            return
        bp.add('cis_unpack_wgrad', self.dwp.data_ptr(), self.wg_kmap.data_ptr(), self.wg_K_pad, min(128, self.cout), self.wg_splits[mode],
               s.ptr(self.wkey, 'grad'), self.colpart.data_ptr(), self.col_blocks[mode], self.cout,
               (self.db_eff.data_ptr() if self.bn else s.ptr(self.bkey, 'grad')), 0 if self.wg_halo else 1)
        for g0, buf in sorted(self.dwp_hi.items()):     # output channels >= 128: dw shifted by g0 (n stride 1)
            if (mode, g0) in self.wg_splits_hi:
                bp.add('cis_unpack_wgrad', buf.data_ptr(), self.wg_kmap.data_ptr(), self.wg_K_pad, min(128, self.cout - g0),
                       self.wg_splits_hi[(mode, g0)], s.ptr(self.wkey, 'grad') + 4 * g0, None, 0, 0, None, 0 if self.wg_halo else 1)
        if self.bn:
            bp.add('cis_bn_chain', s.ptr(self.wkey), s.ptr(self.bkey), s.ptr(self.name + '/gamma'), s.ptr(self.wkey, 'grad'),
                   self.db_eff.data_ptr(), self.k * self.k * self.cin * self.cout, self.cout, s.ptr(self.bkey, 'grad'),
                   s.ptr(self.name + '/gamma', 'grad'), s.ptr(self.name + '/beta', 'grad'))

    # ---- tap tables ------------------------------------------------------------------------------------------
    def fwd_taps(self, H, W):
        pt, _ = same_pad(H, self.k, self.stride, self.dil)
        pl, _ = same_pad(W, self.k, self.stride, self.dil)
        return [(r * self.dil - pt, c * self.dil - pl) for r in range(self.k) for c in range(self.k)], pt, pl

    def setup_wgrad(self, taps, srcs):
        """Weight-gradient kernel path and packed K layout, once: the TMA operand path (8x8 pixel tiles) for stride-1 layers whose concat
        sources are 64-channel aligned, the halo-resident kernel where it fits; both lay the K columns out per tap in 64-channel groups
        and exclude thin inputs (the per-tap 64-channel padding would waste the loads).  Else the gather kernel on the forward K layout."""
        if self.wg_kmap is not None:
            return
        cin8 = len(self.in_chanmap)
        aligned = all(s.C8 % 64 == 0 for s in srcs[:-1])
        self.wg_tma = bool(WGRAD_TMA and self.stride == 1 and cin8 >= 32 and aligned)
        self.wg_halo = bool(WGRAD_HALO and cin8 >= WGRAD_HALO_MIN_CH and wgrad_halo_fits(taps, self.cout, self.stride) and aligned)
        if not (self.wg_tma or self.wg_halo):
            self.wg_K_pad, self.wg_kmap = self.K_pad, self.fwd_kmap
            return
        nch64 = -(-cin8 // 64)
        self.wg_K_pad = ru(self.k * self.k * nch64 * 64, 128)
        km = np.full(self.wg_K_pad, -1, dtype=np.int32)
        fk = self.fwd_kmap.cpu().numpy()
        for t in range(self.k * self.k):
            for pos in range(cin8):
                km[(t * nch64 + pos // 64) * 64 + pos % 64] = fk[t * cin8 + pos]
        self.wg_kmap = torch.from_numpy(km).to(self.device)

    def setup_dgrad(self, H, W):
        """Packed weights for the data gradient on an input of size HxW: one launch for stride 1, four output-parity
        launches for stride 2 (each with the tap subset that lands on that parity)."""
        if self.dgrad_packs is not None:
            return
        _, pt, pl = self.fwd_taps(H, W)
        k, s, d = self.k, self.stride, self.dil
        g_chan = list(range(self.cout)) + [-1] * (ru(self.cout, 8) - self.cout)
        cin8 = len(self.in_chanmap)
        bn_, nt = pick_bn(cin8, self.bn_cap)
        rows = bn_ * nt
        nmap = torch.tensor(list(self.in_chanmap) + [-1] * (rows - cin8), dtype=torch.int32, device=self.device)
        packs = []
        for a in range(s):
            for b in range(s):
                tl, offs = _parity_taps(k, s, d, pt, pl, a, b)
                if not tl:        # k = 1, stride 2: no tap lands on this parity, its input-gradient pixels are zero (see _conv_bwd)
                    packs.append(Pack(a=a, b=b, rows_used=False))
                    continue
                # value = W[t, ci, co] -> flat (t*cin + ci)*cout + co ; K position (ti, co), row n = ci
                kmap, Kp = self._kmap(tl, g_chan, self.cin * self.cout, 1)
                packs.append(Pack(a=a, b=b, taps=offs, kmap=kmap, K_pad=Kp, rows=rows, BN=bn_, n_tiles=nt, nmap=nmap, w=self._rows(rows, Kp)))
        self.dgrad_packs = packs

    def setup_transposed(self, chanmap):
        """tf.layers.conv2d_transpose(k=4, s=2, 'same') as four output-parity stride-1 launches (model_pwcnet.py:286)."""
        assert self.transposed and self.k == 4
        self.in_chanmap = list(chanmap)
        packs = []
        for a in range(2):
            for b in range(2):
                tl, offs = _parity_taps(4, 2, 1, 1, 1, a, b)       # output pixel 2y + a reads input y + dy through tap ky = a + 1 - 2 dy
                # kernel [kh,kw,Cout,Cin]: flat ((t*Cout + co)*Cin + ci) ; K position (ti, ci), row n = co (stride Cin)
                kmap, Kp = self._kmap(tl, chanmap, self.cout * self.cin, 1)
                packs.append(Pack(a=a, b=b, taps=offs, kmap=kmap, K_pad=Kp, rows=self.npad, BN=self.BN, n_tiles=self.n_tiles,
                                  w=self._rows(self.npad, Kp)))
        self.tr_packs = packs

    def setup_transposed_dgrad(self, g_pos):
        """Data gradient of the transposed conv: dx[y, x, ci] = sum dy[2y + ky - 1, 2x + kx - 1, co] * W[ky, kx, co, ci], a 4x4 stride-2
        forward conv of the output gradient.  g_pos: position of output channel co inside the gradient's 8-channel chunk."""
        if self.tr_dgrad is not None:
            return
        g_chan = [-1] * 8
        for co in range(self.cout):
            g_chan[g_pos + co] = co
        cin8 = len(self.in_chanmap)
        bn_, nt = pick_bn(cin8)
        rows = bn_ * nt
        # K position (tap, gradient channel co) -> flat ((t*Cout + co)*Cin), row n -> + ci
        kmap, Kp = self._kmap(range(16), g_chan, self.cout * self.cin, self.cin)
        nmap = torch.tensor(list(self.in_chanmap) + [-1] * (rows - cin8), dtype=torch.int32, device=self.device)
        taps = [(r - 1, c - 1) for r in range(4) for c in range(4)]      # TF 'SAME' k4 s2: one row / column of padding in front
        self.tr_dgrad = Pack(taps=taps, kmap=kmap, K_pad=Kp, rows=rows, BN=bn_, n_tiles=nt, nmap=nmap, w=self._rows(rows, Kp))


def _concat_bwd(bp, mode, srcs, g, nb, OH, OW):
    """Gradient g (nb x OH x OW) of the concat of `srcs` brought to OH x OW -> the sources' gradient slices, ONE launch (the fused
    resize-concat transpose: slices the channels, folds the replicas of batch-broadcast sources, accumulates where a gradient exists)."""
    want = [1 if mode in s.dep else 0 for s in srcs]
    if not any(want):
        return
    garr, acc = [], []
    for s, w in zip(srcs, want):
        if w:
            sg = s.get_grad()
            garr.append(CisSrc(sg.ptr, sg.pitch, sg.c_off, s.C8 // 8, s.n_mod))
            acc.append(1 if s.grad_written.get(mode) else 0)
            s.grad_written[mode] = True
        else:
            garr.append(CisSrc(None, 8, 0, s.C8 // 8, s.n_mod))
            acc.append(0)
    ga = (CisSrc * len(srcs))(*garr)
    wa, aa = (C.c_int32 * len(srcs))(*want), (C.c_int32 * len(srcs))(*acc)
    bp.keep += [ga, wa, aa]
    bp.add('cis_resize_concat_bf16_bwd', g.ptr, g.pitch, g.c_off, nb, OH, OW, ga, wa, aa, len(srcs), srcs[0].H, srcs[0].W)


# ================================================================================================ graph builder
class Builder(object):
    """Builds the forward plan and records backward closures (reverse-mode, hand-scheduled)."""

    def __init__(self, device):
        self.device = device
        self.fwd = Plan('fwd')
        self.lane = 0        # lane given to forward launches (1 = side stream, see Plan.run)
        self.tape = []       # backward closures in forward order
        self.keep = []       # every buffer referenced by raw pointer from a descriptor must outlive the plans

    # ---- helpers
    def new_act(self, N, H, W, C, name='', dep=frozenset(), n_mod=0):
        a = Act(N, H, W, C, self.device, name=name, dep=dep, n_mod=n_mod)
        self.keep.append(a)
        return a

    def hold(self, obj):
        """Register a tensor / Act whose storage is referenced by raw pointer from a launch descriptor."""
        self.keep.append(obj)
        return obj

    def f32(self, *shape):
        return self.hold(torch.zeros(*shape, dtype=torch.float32, device=self.device))

    def _launch(self, plan, d, flops, lane=0):
        """One conv launch, split-K where it pays."""
        setup_splitk(d, self.device, plan.keep)
        plan.keep.append(d)
        plan.add('cis_conv_igemm', C.byref(d), flops=flops, lane=lane)

    def _launch_parities(self, plan, emitted, lane):
        """Output-parity launches [(CisConv, flops)]: ONE grouped launch on `lane` when merge_parity_launches takes them, else one
        launch each on lane 0."""
        grp = merge_parity_launches([d for d, _ in emitted])
        if grp is None:
            for d, fl in emitted:
                self._launch(plan, d, fl)
            return
        plan.keep.append(grp)
        plan.add('cis_conv_igemm', C.byref(grp), flops=sum(f for _, f in emitted), lane=lane)

    def conv(self, layer, srcs, out=None, post_add=None, addf=None, outf=None, outf_ch=0, mode=0, want_bf16=True, name=None,
             plan=None, out_rows=None, grad_out=None):
        """y = act(conv(concat(srcs)) + bias [+ addf]) [+ post_add]; returns the output Act.  grad_out: the Act whose gradient is this
        layer's output gradient (an fp32-only output, want_bf16=False, that feeds the same value as that Act: PWC-Net's flow heads)."""
        plan = plan or self.fwd
        if MATERIALIZE_MISALIGNED_CONCAT and len(srcs) > 1 and layer.tag and layer.stride == 1 and \
                any(s.C8 % 64 for s in srcs[:-1]):
            # materialised concat: the virtual one is not 64-channel aligned, so the TMA operand paths would not apply
            srcs = [self.resize_concat(srcs, name=layer.name + '.cat')]
        s0 = srcs[0]
        N = out_rows or max(s.N for s in srcs)
        H, W = s0.H, s0.W
        for s in srcs:
            assert (s.H, s.W) == (H, W), (layer.name, [(q.H, q.W) for q in srcs])
        chanmap = []
        base = 0
        for s in srcs:
            chanmap += [(m + base if m >= 0 else -1) for m in s.chanmap]
            base += s.C
        if layer.fwd_pack is None:
            layer.setup_fwd(chanmap)
        else:
            assert layer.in_chanmap == chanmap, layer.name
        OH, OW = -(-H // layer.stride), -(-W // layer.stride)
        dep = frozenset().union(*[s.dep for s in srcs]) | ({layer.tag} if layer.tag else frozenset())
        if post_add is not None:
            dep = dep | post_add.dep
        if out is None and want_bf16:
            out = self.new_act(N, OH, OW, layer.cout, name=name or layer.name, dep=dep)
        if out is not None:
            out.dep = out.dep | dep
            gr = [s.gen_rows for s in srcs if s.gen_rows]
            if gr:
                out.gen_rows = gr[0]
        taps, _, _ = layer.fwd_taps(H, W)
        d = conv_desc(N, H, W, OH, OW, layer.stride, taps, [s.src() for s in srcs], layer.fwd_pack, out, bias=layer.bias_ptr(),
                      act=layer.act, alpha=layer.alpha, outf=outf, outf_ch=outf_ch)
        if addf is not None:
            d.addf_pre, d.addf_pitch, d.addf_coff = addf.data_ptr(), addf.shape[-1], 0
            if outf is None:
                d.outf_ch = addf.shape[-1]
        if post_add is not None:
            d.add_post, d.add_post_pitch, d.add_post_coff = post_add.ptr, post_add.pitch, post_add.c_off
        d.mode = mode
        order = setup_halo_s2(d, taps, layer.n_tiles) if (layer.stride == 2 and layer.dil == 1) else None
        layer.place(d, layer.fwd_pack, taps, layer.dil, len(layer.in_chanmap), order)
        plan.keep += [srcs, out, outf, addf, post_add, layer]
        self._launch(plan, d, 2.0 * N * OH * OW * layer.k * layer.k * layer.cin * layer.cout, lane=self.lane)
        if layer.tag:
            # call index: a layer run more than once in one graph (the siamese PWC-Net feature pyramid) gets one range of weight-gradient
            # slices per call, summed by the one un-pack of plan_finalize
            layer.ncalls += 1
            self.tape.append(lambda bp, m, L=layer, S=list(srcs), O=out, P=post_add, K=layer.ncalls - 1, GO=grad_out:
                             self._conv_bwd(bp, m, L, S, O, P, K, GO))
        return out

    def _conv_bwd(self, bp, mode, layer, srcs, out, post_add, call=0, grad_out=None):
        gout = grad_out if grad_out is not None else out
        if gout is None or mode not in gout.dep or not gout.grad_written.get(mode):
            return
        G = gout.get_grad()
        if out is None:
            out = gout            # fp32-only output: no activation (asserted below), the gradient Act gives the row grid
            assert layer.act == ACT_NONE and post_add is None, layer.name
        nb = out.rows(mode)
        npix = nb * out.H * out.W
        if post_add is not None and mode in post_add.dep:
            pg = post_add.get_grad()
            bp.add('cis_add_slice', pg.ptr, pg.pitch, pg.c_off, G.ptr, G.pitch, G.c_off, npix, G.C8 // 8, 1,
                   1 if post_add.grad_written.get(mode) else 0)
            post_add.grad_written[mode] = True
        ncalls = layer.ncalls
        if layer.tag == mode:
            chunks = -(-layer.cout // 8)
            ppb = (256 // chunks) * COLSUM_PIX                      # pixels per colsum block (P pixel lanes x COLSUM_PIX pixels each)
            nblk = max(1, min(592, -(-npix // ppb)))
            layer.col_blocks[mode] = nblk * ncalls                 # call k owns the partial blocks [k * nblk, (k + 1) * nblk)
            if layer.colpart is None:
                layer.colpart = torch.empty(592 * ncalls * layer.cout, dtype=torch.float32, device=self.device)
            colpart = layer.colpart.data_ptr() + 4 * call * nblk * layer.cout
        res = (post_add.ptr, post_add.pitch, post_add.c_off) if post_add is not None else (None, 0, 0)
        fused_colsum = bool(DACT_COLSUM and layer.act != ACT_NONE and layer.tag == mode)
        if fused_colsum:      # activation derivative + bias-gradient partials in one pass over the gradient
            bp.add('cis_dact_colsum', G.ptr, G.pitch, G.c_off, out.ptr, out.pitch, out.c_off, res[0], res[1], res[2], npix, layer.cout,
                   layer.act, layer.alpha, colpart, nblk)
        elif layer.act != ACT_NONE:
            bp.add('cis_dact_mul', G.ptr, G.pitch, G.c_off, out.ptr, out.pitch, out.c_off, res[0], res[1], res[2], npix, G.C8 // 8,
                   layer.act, layer.alpha)
        s0 = srcs[0]
        H, W = s0.H, s0.W
        taps, _, _ = layer.fwd_taps(H, W)
        if layer.tag == mode:   # weight + bias gradients
            layer.setup_wgrad(taps, srcs)
            for g0 in range(0, layer.cout, 128):             # cis_conv_wgrad takes at most 128 output channels
                gc = min(128, layer.cout - g0)
                w = CisWgrad()
                w.N, w.H, w.W, w.OH, w.OW, w.sh, w.sw = nb, H, W, out.H, out.W, layer.stride, layer.stride
                _fill_taps(w, taps)
                _fill_srcs(w, srcs)
                w.g, w.g_pitch, w.g_coff, w.g_chunks = G.ptr, G.pitch, G.c_off + g0, G.C8 // 8 - g0 // 8
                w.Cout, w.K_pad = gc, layer.wg_K_pad
                w.tma = 2 if layer.wg_halo else (1 if layer.wg_tma else 0)
                nkb = (nb * (-(-out.H // 8)) * (-(-out.W // 8))) if w.tma else -(-npix // 64)
                ntile = -(-layer.wg_K_pad // 128)
                if w.tma == 2:      # grid.x = 64-channel chunks of the input, grid.z = tap-pair groups (x 64-channel halves of Cout)
                    w.nh, w.nwg, gz = wgrad_halo_tiling(len(taps), gc)
                    if WGRAD_HALO_NWG < 2:
                        gz = 2 if gc > 64 else 1
                    ntile = (-(-len(layer.in_chanmap) // 64)) * gz
                splits = wgrad_splits(nkb, ntile, gc, layer.wg_K_pad)
                w.splits = splits
                # call k of the layer owns the slices [k * splits, (k + 1) * splits) (every call has the same shape, so the same splits)
                size = splits * ncalls * gc * layer.wg_K_pad
                if g0 == 0:
                    assert ncalls == 1 or layer.wg_splits.get(mode) in (None, splits * ncalls), layer.name
                    layer.wg_splits[mode] = splits * ncalls
                    if layer.dwp is None or layer.dwp.numel() < size:
                        assert not layer.wgrad_modes, 'slice buffer must be sized by the first (largest) mode'
                        layer.dwp = torch.empty(max(layer.wg_splits.values()) * gc * layer.wg_K_pad, dtype=torch.float32, device=self.device)
                    buf = layer.dwp
                else:
                    layer.wg_splits_hi[(mode, g0)] = splits * ncalls
                    if g0 not in layer.dwp_hi or layer.dwp_hi[g0].numel() < size:
                        assert not layer.wgrad_modes, 'slice buffer must be sized by the first (largest) mode'
                        layer.dwp_hi[g0] = torch.empty(size, dtype=torch.float32, device=self.device)
                    buf = layer.dwp_hi[g0]
                w.dwp = buf.data_ptr() + 4 * call * splits * gc * layer.wg_K_pad
                bp.keep.append(w)
                bp.add('cis_conv_wgrad', C.byref(w), flops=2.0 * npix * layer.k * layer.k * layer.cin * gc, lane=1)
            layer.wgrad_modes.add(mode)
            if not fused_colsum:
                bp.add('cis_colsum', G.ptr, G.pitch, G.c_off, npix, layer.cout, colpart, nblk, lane=1)
        need = [s for s in srcs if mode in s.dep]
        if not need:
            return
        layer.setup_dgrad(H, W)
        layer.dgrad_used = True
        cin8 = len(layer.in_chanmap)
        single = (len(srcs) == 1 and srcs[0].n_mod == 0)
        if single:
            tgt = srcs[0].get_grad()
            acc = bool(srcs[0].grad_written.get(mode))
        else:
            if layer.dcat is None:
                layer.dcat = Act(max(s.N for s in srcs), H, W, cin8, self.device, chanmap=layer.in_chanmap, name=layer.name + '.dcat')
            tgt, acc = layer.dcat, False
        if not acc and any(not pk.taps for pk in layer.dgrad_packs):
            # a parity no tap reaches (k = 1, stride 2) contributes nothing: when accumulating its pixels keep what they hold, on the
            # first write they are zero -- zero the whole slice (add_slice of 0 sources), the parities with taps then overwrite theirs
            bp.add('cis_add_slice', tgt.ptr, tgt.pitch, tgt.c_off, tgt.ptr, tgt.pitch, tgt.c_off, nb * H * W, tgt.C8 // 8, 0, 0)
        emitted = []
        s = layer.stride
        for pk in layer.dgrad_packs:
            oh = -(-(H - pk.a) // s)
            ow = -(-(W - pk.b) // s)
            if oh <= 0 or ow <= 0 or not pk.taps:
                continue
            d = conv_desc(nb, out.H, out.W, oh, ow, 1, pk.taps, [G.src()], pk, tgt, grid=(H, W, s, pk.a, pk.b), add_pre=acc)
            layer.place(d, pk, pk.taps, layer.dil if s == 1 else 1, ru(layer.cout, 8))
            emitted.append((d, 2.0 * nb * oh * ow * len(pk.taps) * layer.cin * layer.cout))
        self._launch_parities(bp, emitted, lane=0)
        if single:
            srcs[0].grad_written[mode] = True
        else:
            _concat_bwd(bp, mode, srcs, tgt, nb, H, W)     # the virtual concat's gradient -> the sources' gradient slices

    # ---- fused resize + concat: ONE launch brings up to 4 same-resolution sources (batch-broadcast ones included) to OH x OW and lays
    # them side by side in one buffer, ONE launch takes the gradient back (folding the broadcast replicas); replaces a resize launch
    # per source plus a copy per source and replica (recover decoder: `deconv` inputs, nets.py:80-104; misaligned virtual concats)
    def resize_concat(self, srcs, OH=None, OW=None, name='cat'):
        srcs = list(srcs)
        assert 1 <= len(srcs) <= 4
        N = max(s.N for s in srcs)
        H, W = srcs[0].H, srcs[0].W
        OH, OW = OH or H, OW or W
        for s in srcs:
            assert (s.H, s.W) == (H, W) and (s.n_mod == 0 or N % s.n_mod == 0)
        chanmap, base = [], 0
        for s in srcs:
            chanmap += [(m + base if m >= 0 else -1) for m in s.chanmap]
            base += s.C
        dep = frozenset().union(*[s.dep for s in srcs])
        cat = Act(N, OH, OW, base, self.device, chanmap=chanmap, dep=dep, name=name)
        gr = [s.gen_rows for s in srcs if s.gen_rows]
        if gr:
            cat.gen_rows = gr[0]
        arr = (CisSrc * len(srcs))(*[s.src() for s in srcs])
        self.keep += [srcs, cat, arr]
        self.fwd.add('cis_resize_concat_bf16', arr, len(srcs), N, H, W, cat.ptr, cat.pitch, cat.c_off, OH, OW, lane=self.lane)

        def bwd(bp, mode):
            if mode not in cat.dep or not cat.grad_written.get(mode):
                return
            _concat_bwd(bp, mode, srcs, cat.get_grad(), cat.rows(mode), OH, OW)
        self.tape.append(bwd)
        return cat

    # ---- transposed conv (PWC-Net up_flow / up_feat)
    def conv_transpose(self, layer, src, out=None, outf=None, plan=None, name=None):
        plan = plan or self.fwd
        if layer.tr_packs is None:
            layer.setup_transposed(src.chanmap)
        N, H, W = src.N, src.H, src.W
        if out is None:
            out = self.new_act(N, 2 * H, 2 * W, layer.cout, name=name or layer.name, dep=src.dep)
        if layer.tag:
            out.dep = out.dep | src.dep | {layer.tag}
            self.tape.append(lambda bp, m, L=layer, S=src, O=out: self._conv_transpose_bwd(bp, m, L, S, O))
        emitted = []
        for pk in layer.tr_packs:
            d = conv_desc(N, H, W, H, W, 1, pk.taps, [src.src()], pk, out, out_ch=layer.cout, bias=layer.bias_ptr(),
                          grid=(2 * H, 2 * W, 2, pk.a, pk.b), outf=outf, outf_ch=layer.cout)
            layer.place(d, pk, pk.taps, 1, len(layer.in_chanmap))
            emitted.append((d, 2.0 * N * H * W * len(pk.taps) * layer.cin * layer.cout))
        plan.keep += [src, out, outf, layer]
        self._launch_parities(plan, emitted, lane=self.lane)
        return out

    def _conv_transpose_bwd(self, bp, mode, layer, src, out):
        """Backward of conv_transpose.  Weights: the output gradient is split into its four output-parity planes, and parity (a, b) is a
        stride-1 weight gradient over the taps setup_transposed gives it (gather kernel, private slices per parity, one un-pack job each);
        bias: column sums over the four planes.  Data: a 4x4 stride-2 forward conv of the output gradient (setup_transposed_dgrad)."""
        if mode not in out.dep or not out.grad_written.get(mode):
            return
        G = out.get_grad()
        N, h, w = src.N, src.H, src.W
        npix = N * h * w
        if layer.tag == mode:
            if layer.tr_planes is None:
                layer.tr_planes = torch.zeros(4, N, h, w, 8, dtype=torch.bfloat16, device=self.device)
                layer.colpart = torch.empty(592 * layer.cout, dtype=torch.float32, device=self.device)
            planes = layer.tr_planes
            bp.add('cis_parity_split_bf16', G.ptr, G.pitch, G.c_off, N, h, w, layer.cout, planes.data_ptr(), 8)
            layer.col_blocks[mode] = max(1, min(592, -(-4 * npix // (256 * COLSUM_PIX))))
            bp.add('cis_colsum', planes.data_ptr(), 8, 0, 4 * npix, layer.cout, layer.colpart.data_ptr(), layer.col_blocks[mode], lane=1)
            for q, pk in enumerate(layer.tr_packs):
                wg = CisWgrad()
                wg.N, wg.H, wg.W, wg.OH, wg.OW, wg.sh, wg.sw = N, h, w, h, w, 1, 1
                _fill_taps(wg, pk.taps)
                _fill_srcs(wg, [src])
                wg.g, wg.g_pitch, wg.g_coff, wg.g_chunks = planes[q].data_ptr(), 8, 0, 1
                wg.Cout, wg.K_pad, wg.tma = layer.cout, pk.K_pad, 0
                nkb = -(-npix // 64)
                wg.splits = wgrad_splits(nkb, -(-pk.K_pad // 128), layer.cout, pk.K_pad)
                pk.wg_splits[mode] = wg.splits
                if pk.dwp is None or pk.dwp.numel() < wg.splits * layer.cout * pk.K_pad:
                    pk.dwp = torch.empty(wg.splits * layer.cout * pk.K_pad, dtype=torch.float32, device=self.device)
                wg.dwp = pk.dwp.data_ptr()
                bp.keep.append(wg)
                bp.add('cis_conv_wgrad', C.byref(wg), flops=2.0 * npix * len(pk.taps) * layer.cin * layer.cout, lane=1)
        if mode not in src.dep:
            return
        g_pos = G.c_off % 8                  # the gradient's channels inside its 8-channel chunk (up_feat sits behind up_flow)
        layer.setup_transposed_dgrad(g_pos)
        dg, tgt = layer.tr_dgrad, src.get_grad()
        d = conv_desc(N, 2 * h, 2 * w, h, w, 2, dg.taps, [CisSrc(G.ptr, G.pitch, G.c_off - g_pos, 1, 0)], dg, tgt,
                      add_pre=bool(src.grad_written.get(mode)))
        self._launch(bp, d, 2.0 * npix * 16 * layer.cin * layer.cout)
        src.grad_written[mode] = True

    # ---- resampling ops
    def resize_bilinear(self, src, OH, OW, name=''):
        """tf.image.resize_images legacy bilinear (convolution_utils.py:88); identity when the size matches."""
        if (src.H, src.W) == (OH, OW):
            return src
        out = Act(src.N, OH, OW, src.C, self.device, chanmap=src.chanmap, n_mod=src.n_mod, dep=src.dep, name=name or src.name + '.rs')
        out.gen_rows = src.gen_rows
        self.keep += [src, out]
        self.fwd.add('cis_resize_bilinear_bf16', src.ptr, src.pitch, src.c_off, src.N, src.H, src.W, out.ptr, out.pitch, out.c_off, OH, OW,
                     src.C8 // 8)

        def bwd(bp, mode):
            if mode not in out.dep or not out.grad_written.get(mode):
                return
            g, sg = out.get_grad(), src.get_grad()
            bp.add('cis_resize_bilinear_bf16_bwd', g.ptr, g.pitch, g.c_off, out.rows(mode), OH, OW, sg.ptr, sg.pitch, sg.c_off, src.H, src.W,
                   src.C8 // 8, 1 if src.grad_written.get(mode) else 0)
            src.grad_written[mode] = True
        self.tape.append(bwd)
        return out

    def upsample_nn2x(self, src, name=''):
        """tf.image.resize_nearest_neighbor(align_corners=True) x2 (convolution_utils.py:71)."""
        assert src.c_off == 0 and src.pitch == src.C8
        out = Act(src.N, 2 * src.H, 2 * src.W, src.C, self.device, chanmap=src.chanmap, dep=src.dep, name=name or src.name + '.up')
        self.keep += [src, out]
        self.fwd.add('cis_upsample_nn2x', src.ptr, src.N, src.H, src.W, src.pitch, out.ptr)

        def bwd(bp, mode):
            if mode not in out.dep or not out.grad_written.get(mode):
                return
            g, sg = out.get_grad(), src.get_grad()
            bp.add('cis_upsample_nn2x_bwd', g.ptr, src.N, src.H, src.W, src.pitch, sg.ptr, 1 if src.grad_written.get(mode) else 0)
            src.grad_written[mode] = True
        self.tape.append(bwd)
        return out

    def build_backward(self, mode, seeds):
        """seeds: Acts whose .grad has been written by the loss backward.  Returns the backward Plan for `mode`."""
        bp = Plan('bwd_' + mode)
        for a in seeds:
            a.grad_written[mode] = True
        for fn in reversed(self.tape):
            fn(bp, mode)
        return bp

    def backward_plan(self, mode, seed, seeds, layers):
        """The backward Plan of `mode`: the Plan `seed` (the launches that write the gradients of the Acts `seeds`), the reverse tape, a
        join of the weight-gradient lane, then the fixed-order reduction of the weight-gradient slices and the BN chain rule of `layers`
        (one cis_param_multi launch per kind)."""
        full = Plan('bwd_' + mode)
        full.extend(seed)
        full.extend(self.build_backward(mode, seeds))
        full.join()
        fin = Plan('fin_' + mode)
        for L in layers:
            L.plan_finalize(fin, mode)
        full.extend(fin.batch_param_ops(self.device))
        return full
