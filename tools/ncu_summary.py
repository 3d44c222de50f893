"""Summarise an .ncu-rep (raw + source pages) for one kernel: key metrics, stall mix,
instruction hot spots.  Usage: python tools/ncu_summary.py build/prof.ncu-rep [lo hi]
NCU_KERNEL=<regex> picks the kernel when the report holds several."""
import csv
import io
import os
import subprocess
import sys


def page(rep, name):
    sel = ["-k", "regex:" + os.environ["NCU_KERNEL"]] if os.environ.get("NCU_KERNEL") else []
    out = subprocess.run(["ncu", "-i", rep] + sel + ["--page", name, "--csv"], capture_output=True, text=True).stdout
    return list(csv.reader(io.StringIO(out)))


def main():
    rep = sys.argv[1]
    rows = page(rep, "raw")
    hdr, units, vals = rows[0], rows[1], rows[2]
    want = ['gpu__time_duration.sum', 'dram__bytes_read.sum', 'dram__bytes_write.sum',
            'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed', 'sm__warps_active.avg.pct_of_peak_sustained_active',
            'launch__registers_per_thread', 'launch__occupancy_limit_shared_mem', 'launch__grid_size',
            'smsp__issue_active.avg.pct_of_peak_sustained_active', 'smsp__inst_executed.sum',
            'l1tex__data_pipe_lsu_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed',
            'sm__cycles_elapsed.max', 'launch__shared_mem_per_block_dynamic', 'lts__t_sectors_op_write.sum',
            'l1tex__data_bank_conflicts_pipe_lsu_mem_shared_op_st.sum', 'smsp__warps_eligible.avg.per_cycle_active']
    for h, u, v in zip(hdr, units, vals):
        if h in want:
            print(f"{h:75s} {u:12s} {v}")
    rows = page(rep, "source")
    hdr = rows[1]
    data = []
    for r in rows[2:]:   # a report with several launches repeats the table: first launch only
        if len(r) < len(hdr) or not r[hdr.index('# Samples')].isdigit():
            break
        data.append(r)
    isrc = hdr.index('Source'); isamp = hdr.index('# Samples'); iinst = hdr.index('Instructions Executed')
    tot_s = sum(int(r[isamp]) for r in data); tot_i = sum(int(r[iinst]) for r in data)
    print('total samples', tot_s, 'total warp-inst', tot_i)
    stalls = [h for h in hdr if h.startswith('stall_') and 'Not Issued' not in h]
    agg = {s: sum(int(r[hdr.index(s)]) for r in data) for s in stalls}
    print('stall mix:', ', '.join(f"{k[6:]}={v * 100 // max(tot_s, 1)}%" for k, v in sorted(agg.items(), key=lambda kv: -kv[1])[:9]))
    groups = []
    for i, r in enumerate(data):
        c = int(r[iinst])
        if groups and groups[-1]['c'] == c:
            g = groups[-1]; g['n'] += 1; g['samp'] += int(r[isamp]); g['end'] = i
        else:
            groups.append({'c': c, 'n': 1, 'samp': int(r[isamp]), 'start': i, 'end': i})
    print('regions (>=1% of instructions or samples):')
    for g in groups:
        if g['c'] * g['n'] > tot_i * 0.01 or g['samp'] > tot_s * 0.01:
            print(f"  sass[{g['start']:4d}-{g['end']:4d}] execs={g['c']:9d} x{g['n']:3d} = {g['c'] * g['n'] * 100 / tot_i:5.1f}% inst, "
                  f"{g['samp'] * 100 / tot_s:5.1f}% samples   {data[g['start']][isrc][:44]}")
    if len(sys.argv) > 2:
        lo, hi = int(sys.argv[2]), int(sys.argv[3])
        for i in range(lo, hi + 1):
            r = data[i]
            st = {s[6:]: int(r[hdr.index(s)]) for s in stalls if int(r[hdr.index(s)]) > 0}
            print(i, r[isrc][:60].ljust(60), r[iinst], r[isamp], st)


if __name__ == "__main__":
    main()
