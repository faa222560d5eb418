"""Offline launch-plan report (no GPU needed: the step graph is BUILT on CPU tensors, nothing is launched).
For every conv launch of the forward / backward plans: kernel family, tile shape, CTA count, serial pipeline steps per CTA, and which
of the prepared experiment switches (DESIGN.md section 6) would touch it.  Honours the same environment switches as the engine,
e.g.  CIS_SPLITK=2 CIS_SPLITK_MAX=16 CIS_SPLITK_NCTA=8 CIS_SPLITK_MIN_UNITS=32 python tools/plan_report.py"""
import collections
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from unsupervised_detection_b200 import engine  # noqa: E402
from unsupervised_detection_b200.step_graph import CISGraph  # noqa: E402


def conv_row(d):
    chunks = sum(d.src[i].chunks for i in range(d.nsrc))
    if d.halo:
        dd = d.dil
        hp0, wp0 = -(-d.OH // dd), -(-d.OW // dd)
        mtc = d.MT * max(d.nwg, 1)          # 16x8 tiles per CTA (nwg MMA warpgroups of MT tiles each)
        tiles = (-(-wp0 // 8)) * (-(-hp0 // (16 * mtc))) * dd * dd * d.N
        nchunks = -(-chunks // 8)
        steps = nchunks * d.ntaps
        kind = 'halo'
        wtile = d.BN * 128
    else:
        tiles = -(-(d.N * d.OH * d.OW) // 128)
        steps = d.K_pad // 64
        kind = 'gen'
        wtile = d.BN * 128
    splits = max(1, d.splits)
    ncta = tiles * d.n_tiles * splits
    return dict(kind=kind, BN=d.BN, nt=d.n_tiles, MT=d.MT if d.halo else 1, nwg=max(d.nwg, 1) if d.halo else 1, N=d.N, OH=d.OH, OW=d.OW, taps=d.ntaps, cin=chunks * 8,
                tiles=tiles, ncta=ncta, steps=-(-steps // splits), splits=splits, two_launch=bool(splits > 1 and not d.sk_counters),
                ws_fit=bool(d.halo and d.dil == 1 and d.n_tiles == 1 and d.BN <= 32 and steps >= 2 and
                            2 * (((8 + d.ex) * (16 * mtc + d.ey) * 128 + 1023) // 1024 * 1024) + 1024 + steps * wtile <= 200 * 1024),
                cluster=bool(d.halo and d.BN >= 64 and (tiles % 2 == 0)))


def main():
    H, W, B = int(os.environ.get('PLAN_H', 256)), int(os.environ.get('PLAN_W', 448)), int(os.environ.get('PLAN_B', 4))
    g = CISGraph(H, W, B, device='cpu', global_batch=B)
    rows = []
    for pname, plan, w in (('fwd', g.fwd, 4), ('bwdG', g.bwd['G'], 3), ('bwdR', g.bwd['R'], 1)):
        for fn, a, name, fl, lane in plan.ops:
            if name == 'cis_conv_igemm':
                r = conv_row(a[0]._obj)
                r.update(plan=pname, w=w, flops=fl)
                rows.append(r)
    print('%d conv launches in the three plans; per step (1R:3G): %.1f' % (len(rows), sum(r['w'] for r in rows) / 4.0))
    print('%-5s %-4s %4s %3s %3s %3s %3s %9s %5s %6s %6s %6s %6s  %s' % ('plan', 'kern', 'BN', 'nt', 'MT', 'nwg', 'N', 'OHxOW', 'taps', 'cin', 'CTAs',
                                                                  'steps', 'split', 'flags'))
    for r in sorted(rows, key=lambda r: (r['ncta'], -r['steps'])):
        flags = ' '.join(k for k in ('two_launch', 'ws_fit', 'cluster') if r[k])
        print('%-5s %-4s %4d %3d %3d %3d %3d %4dx%-4d %5d %6d %6d %6d %6d  %s' % (r['plan'], r['kind'], r['BN'], r['nt'], r['MT'], r['nwg'], r['N'], r['OH'],
                                                                           r['OW'], r['taps'], r['cin'], r['ncta'], r['steps'], r['splits'], flags))
    few = [r for r in rows if r['ncta'] <= 32]
    print('\nlaunches with <= 32 CTAs: %.1f per step, serial steps per CTA: median %d, max %d' %
          (sum(r['w'] for r in few) / 4.0, sorted(r['steps'] for r in few)[len(few) // 2] if few else 0, max([r['steps'] for r in few] or [0])))
    hist = collections.Counter()
    for r in rows:
        b = 1 if r['ncta'] <= 8 else 2 if r['ncta'] <= 32 else 3 if r['ncta'] <= 148 else 4 if r['ncta'] <= 592 else 5
        hist[b] += r['w'] / 4.0
    print('launches per step by CTA count: <=8: %.1f | 9-32: %.1f | 33-148: %.1f | 149-592: %.1f | >592: %.1f' % tuple(hist[i] for i in range(1, 6)))
    print('weight-stationary-eligible (CIS_PERSIST_WS): %.1f per step; cluster-eligible (CIS_HALO_CLUSTER=2): %.1f per step; split: %.1f per step' %
          (sum(r['w'] for r in rows if r['ws_fit']) / 4.0, sum(r['w'] for r in rows if r['cluster']) / 4.0, sum(r['w'] for r in rows if r['splits'] > 1) / 4.0))
    wgrad_report(g)


def wgrad_report(g):
    """Halo weight-gradient launches (CisWgrad.tma = 2): MMA N, MMA warpgroups, grid, and issued / useful MMA work per step."""
    print('\nhalo wgrad launches (tma = 2)')
    print('%-5s %3s %9s %5s %5s %5s %3s %3s %14s  %s' % ('plan', 'N', 'OHxOW', 'taps', 'cin', 'cout', 'nh', 'nwg', 'grid', 'GFLOP issued/useful'))
    useful = issued = 0.0
    for pname, plan, w in (('bwdG', g.bwd['G'], 3), ('bwdR', g.bwd['R'], 1)):
        for fn, a, name, fl, lane in plan.ops:
            if name != 'cis_conv_wgrad' or a[0]._obj.tma != 2:
                continue
            d = a[0]._obj
            chunks = sum(d.src[i].chunks for i in range(d.nsrc))
            nch64 = -(-chunks // 8)
            nh, nwg, gz = d.nh or 64, max(d.nwg, 1), engine.wgrad_halo_tiling(d.ntaps, d.Cout)[2]
            nblk = d.N * (-(-d.OH // 8)) * (-(-d.OW // 8))
            # every CTA row of pairs along grid.z issues its real pairs; Cout > 64 on one warpgroup repeats them per Cout half
            pairs = (d.ntaps + 1) // 2 * (2 if d.Cout > 64 else 1)
            iss = nblk * nch64 * pairs * 2.0 * 128 * nh * 64
            use = 2.0 * d.N * d.OH * d.OW * d.ntaps * chunks * 8 * d.Cout
            useful += w * use / 4.0
            issued += w * iss / 4.0
            print('%-5s %3d %4dx%-4d %5d %5d %5d %3d %3d %14s  %.1f / %.1f' % (pname, d.N, d.OH, d.OW, d.ntaps, chunks * 8, d.Cout, nh, nwg,
                                                                       '%dx%dx%d' % (nch64, d.splits, gz), iss / 1e9, use / 1e9))
    if useful:
        print('per step (1R:3G): %.1f GFLOP issued for %.1f useful (%.2fx)' % (issued / 1e9, useful / 1e9, issued / useful))


if __name__ == '__main__':
    main()
