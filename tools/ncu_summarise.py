"""Summarise `ncu --set full` reports into one JSON.

  python tools/ncu_summarise.py REPORT_DIR > ncu_full_summary.json

For every *.ncu-rep in the directory: one record per captured launch with the metrics the roofline discussion uses (duration, DRAM bytes,
tensor-pipe and tensor-operand shared-memory pipe utilisation, L2 / L1 throughput, occupancy limits)."""
import csv
import io
import json
import os
import subprocess
import sys

KEEP = ['Kernel Name', 'Block Size', 'Grid Size', 'gpu__time_duration.sum', 'dram__bytes_read.sum', 'dram__bytes_write.sum',
        'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed', 'lts__throughput.avg.pct_of_peak_sustained_elapsed',
        'l1tex__throughput.avg.pct_of_peak_sustained_active', 'l1tex__data_bank_reads.avg.pct_of_peak_sustained_elapsed',
        'l1tex__data_bank_writes.avg.pct_of_peak_sustained_elapsed',
        'l1tex__data_pipe_tc_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed',
        'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active', 'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed',
        'sm__throughput.avg.pct_of_peak_sustained_elapsed', 'sm__warps_active.avg.pct_of_peak_sustained_active', 'smsp__cycles_active.avg',
        'launch__registers_per_thread', 'launch__shared_mem_per_block_dynamic', 'launch__occupancy_limit_shared_mem',
        'launch__occupancy_limit_registers', 'launch__waves_per_multiprocessor', 'sm__cycles_elapsed.max']


def summarise(path):
    out = subprocess.run(['ncu', '-i', path, '--page', 'raw', '--csv'], capture_output=True, text=True).stdout
    lines = [l for l in out.splitlines() if l.startswith('"')]
    if len(lines) < 3:
        return []
    rows = list(csv.reader(io.StringIO('\n'.join(lines))))
    head, units, body = rows[0], rows[1], rows[2:]
    recs = []
    for r in body:
        d = {}
        for k in KEEP:
            if k in head:
                i = head.index(k)
                d[k] = (r[i] + ' ' + units[i]).strip() if units[i] else r[i]
        recs.append(d)
    return recs


if __name__ == '__main__':
    root = sys.argv[1]
    res = {}
    for f in sorted(os.listdir(root)):
        if f.endswith('.ncu-rep'):
            res[f[:-8]] = summarise(os.path.join(root, f))
    json.dump(res, sys.stdout, indent=1)
