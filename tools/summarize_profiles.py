"""Nsight Compute raw CSV exports (`ncu --page raw --csv`) -> compact per-launch tables under profiles/ (not kept in git).

usage: python tools/summarize_profiles.py r01
Keeps, per profiled launch: kernel, grid, duration, DRAM bytes read/written, DRAM / L1 / L2 / SM throughput %, occupancy, registers.
The full reports are large; these tables are what a roofline analysis of the kernels needs.
"""
import csv
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEEP = [('gpu__time_duration.sum', 'duration_us'), ('dram__bytes_read.sum', 'dram_read_MB'), ('dram__bytes_write.sum', 'dram_write_MB'),
        ('gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed', 'dram_pct'), ('lts__throughput.avg.pct_of_peak_sustained_elapsed', 'l2_pct'),
        ('l1tex__throughput.avg.pct_of_peak_sustained_active', 'l1_pct'), ('sm__throughput.avg.pct_of_peak_sustained_elapsed', 'sm_pct'),
        ('sm__warps_active.avg.pct_of_peak_sustained_active', 'occupancy_pct'), ('launch__registers_per_thread', 'registers'),
        # tensor pipe: what the north star asks the captures to report next to the HBM numbers (`--set full` collects the first two; the explicit
        # --metrics pass of tools/gpu_profile_r2.sh adds the others where the tool exposes them for sm_100)
        ('TPC.TriageCompute.sm__pipe_tensor_cycles_active_realtime.avg.pct_of_peak_sustained_elapsed', 'tensor_pipe_pct'),
        ('sm__inst_executed_pipe_tensor.sum', 'tensor_inst'),
        ('sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active', 'tensor_pipe_active_pct'),
        ('dram__throughput.avg.pct_of_peak_sustained_elapsed', 'dram_throughput_pct')]
SCALE = {'ns': 1e-3, 'us': 1.0, 'ms': 1e3, 'byte': 1e-6, 'Kbyte': 1e-3, 'Mbyte': 1.0, 'Gbyte': 1e3}


def summarize(src, dst):
    rows = list(csv.reader(open(src)))
    hdr, units, data = rows[0], rows[1], rows[2:]
    H = {h: i for i, h in enumerate(hdr)}
    out = [['id', 'kernel', 'grid', 'block'] + [k for _, k in KEEP]]
    for i, r in enumerate(data):
        name = re.sub(r'\(.*', '', r[H['Kernel Name']]).replace('void ', '').replace('sfb::', '')
        rec = [i, name, r[H['Grid Size']], r[H['Block Size']]]
        for col, _ in KEEP:
            try:
                v = float(r[H[col]].replace(',', '')) if col in H and r[H[col]] not in ('', 'n/a') else float('nan')
            except ValueError:
                v = float('nan')
            v *= SCALE.get(units[H[col]], 1.0) if col in H else 1.0
            rec.append(round(v, 3))
        out.append(rec)
    csv.writer(open(dst, 'w')).writerows(out)
    return out


if __name__ == '__main__':
    tag = sys.argv[1] if len(sys.argv) > 1 else 'r01'
    go = os.path.join(ROOT, 'gpurun_out')
    stems = [a for a in sys.argv[2:]] or ['conv_full', 'render_full']
    for stem in stems:
        src = os.path.join(go, stem + '_raw.csv')
        if os.path.exists(src):
            t = summarize(src, os.path.join(ROOT, 'profiles', f'{tag}_{stem}_ncu.csv'))
            dur = sum(r[4] for r in t[1:])
            rd = sum(r[5] for r in t[1:])
            print(f'{stem}: {len(t) - 1} launches, {dur:.1f} us summed, {rd:.1f} MB DRAM read')
