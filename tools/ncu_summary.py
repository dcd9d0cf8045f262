"""Summarise an .ncu-rep (raw page) + a launch-list csv into markdown / json."""
import csv, json, subprocess, sys
from collections import defaultdict

WANT = ['gpu__time_duration.sum', 'dram__bytes_read.sum', 'dram__bytes_write.sum',
        'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed',
        'sm__warps_active.avg.pct_of_peak_sustained_active', 'launch__registers_per_thread',
        'launch__grid_size', 'launch__block_size', 'launch__occupancy_limit_registers',
        'sm__throughput.avg.pct_of_peak_sustained_elapsed',
        'smsp__issue_active.avg.pct_of_peak_sustained_active',
        'sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active',
        'sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active',
        'sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active',
        'smsp__inst_executed.sum', 'launch__waves_per_multiprocessor',
        'lts__t_sector_hit_rate.pct', 'l1tex__t_sector_hit_rate.pct',
        'smsp__pcsamp_warps_issue_stalled_long_scoreboard', 'smsp__pcsamp_sample_buffer_full']


def rep(path):
    out = subprocess.run(['ncu', '-i', path, '--page', 'raw', '--csv'], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units = rows[0], rows[1]
    res = []
    for r in rows[2:]:
        d = {'kernel': r[hdr.index('Kernel Name')]}
        for w in WANT:
            if w in hdr:
                d[w] = (r[hdr.index(w)], units[hdr.index(w)])
        res.append(d)
    return res


def launches(path):
    rows = [r for r in csv.reader(open(path)) if len(r) > 5]
    hdr = rows[0]
    ki, vi = hdr.index('Kernel Name'), hdr.index('Metric Value')
    agg = defaultdict(list)
    for r in rows[1:]:
        try:
            agg[r[ki].split('(')[0]].append(float(r[vi].replace(',', '')))
        except ValueError:
            pass
    return agg


if __name__ == '__main__':
    kind, path = sys.argv[1], sys.argv[2]
    if kind == 'rep':
        for d in rep(path):
            print('##', d.pop('kernel')[:80])
            for k, (v, u) in d.items():
                print('- %s = %s %s' % (k, v, u))
    else:
        agg = launches(path)
        tot = sum(sum(v) for v in agg.values())
        print('| kernel | launches | avg us | share |\n|---|---|---|---|')
        for k, v in sorted(agg.items(), key=lambda kv: -sum(kv[1])):
            print('| %s | %d | %.1f | %.1f%% |' % (k, len(v), sum(v) / len(v) / 1e3, 100 * sum(v) / tot))
