"""Register occupancy of the convolution kernels, read from the built library (cuobjdump --dump-resource-usage; no GPU needed).

The one-MMA-warpgroup halo kernels and the gather kernels' CPS = 2 instances (BN <= 64) run two CTAs per SM, so that one CTA's prologue and
epilogue overlap the other's main loop: two of them must fit the SM's 65,536 registers, i.e. REG (allocated in units of 8 per thread)
x threads <= 32,768, without local memory.  Where warpgroups re-balance registers with setmaxnreg, the CTA must own at least the sum of
the per-warpgroup budgets, or setmaxnreg.inc would wait forever."""
import re
import shutil
import os
import subprocess

import pytest

from unsupervised_detection_b200 import _lib

# mangled instance -> (threads per CTA, per-warpgroup setmaxnreg budgets of the main loop, or None)
TWO_PER_SM = {
    '_ZN3cis16conv_halo_kernelILi16ELi1EEEv7CisConviiiNS_8HaloMapsEii': (256, None),
    '_ZN3cis16conv_halo_kernelILi32ELi1EEEv7CisConviiiNS_8HaloMapsEii': (256, (88, 168)),
    '_ZN3cis16conv_halo_kernelILi64ELi1EEEv7CisConviiiNS_8HaloMapsEii': (256, (88, 168)),
    '_ZN3cis16conv_halo_kernelILi128ELi1EEEv7CisConviiiNS_8HaloMapsEii': (256, (88, 168)),
    '_ZN3cis17conv_igemm_kernelILi16ELi2EEEv7CisConv': (384, None),
    '_ZN3cis17conv_igemm_kernelILi32ELi2EEEv7CisConv': (384, None),
    '_ZN3cis17conv_igemm_kernelILi64ELi2EEEv7CisConv': (384, (72, 72, 96)),
}


def _cuobjdump():
    exe = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(exe):
        pytest.skip('cuobjdump not installed')
    return exe


def _resource_usage(path):
    out, cur = {}, None
    for line in subprocess.check_output([_cuobjdump(), '--dump-resource-usage', path], text=True).splitlines():
        m = re.match(r'\s*Function (\S+):', line)
        if m:
            cur = m.group(1)
            continue
        if cur is not None and 'REG:' in line:
            out[cur] = {k: int(v) for k, v in re.findall(r'(\w+):(\d+)', line)}
            cur = None
    return out


def _sass(path, fn):
    return subprocess.check_output([_cuobjdump(), '-sass', '-fun', fn, path], text=True)


@pytest.mark.parametrize('fn', sorted(TWO_PER_SM))
def test_two_ctas_per_sm_fit_the_register_file(fn):
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip('library not built')
    use = _resource_usage(_lib.LIB_PATH)
    assert fn in use, 'kernel instance missing from the library: %s' % fn
    r = use[fn]
    threads, budgets = TWO_PER_SM[fn]
    regs = -(-r['REG'] // 8) * 8
    assert regs * threads <= 32768, '%s: %d registers x %d threads' % (fn, r['REG'], threads)
    assert r['LOCAL'] == 0 and r['STACK'] == 0, '%s spills: %s' % (fn, r)
    setmax = re.findall(r'USETMAXREG\.(\w+)\.CTAPOOL[^,;]*?,?\s*(0x[0-9a-f]+)\s*;', _sass(_lib.LIB_PATH, fn))
    if budgets is None:
        assert not setmax, '%s: unexpected setmaxnreg %s' % (fn, setmax)
        return
    # the CTA's pool (threads x REG) covers every warpgroup's budget at once, and setmaxnreg was not dropped by the compiler
    assert 128 * sum(budgets) <= threads * r['REG'], '%s: pool %d < %d' % (fn, threads * r['REG'], 128 * sum(budgets))
    counts = {int(v, 16) for _, v in setmax}
    assert set(budgets) <= counts and r['REG'] in counts, '%s: setmaxnreg counts %s' % (fn, sorted(counts))
