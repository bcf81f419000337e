"""Condenses an `ncu --page raw --csv` dump into one line per launch: kernel, grid, duration, DRAM bytes, DRAM / tensor-pipe
utilisation, achieved occupancy, registers — the per-kernel evidence table.
    ncu -i tools_out/kernels.ncu-rep --page raw --csv > raw.csv ; python tools/ncu_summarize.py raw.csv > tools_out/ncu_kernels.txt"""
import csv
import sys

rows = list(csv.reader(l for l in open(sys.argv[1]) if l.startswith('"')))      # (ncu's ==PROF== banner lines precede the table)
hdr = rows[0]
units = rows[1]
want = {
    'name': 'Kernel Name', 'grid': 'Grid Size', 'block': 'Block Size', 'dur': 'gpu__time_duration.sum',
    'rd': 'dram__bytes_read.sum', 'wr': 'dram__bytes_write.sum', 'dram_pct': 'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed',
    'tensor_pct': 'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active', 'tensor_pct2': 'sm__inst_executed_pipe_tensor.avg.pct_of_peak_sustained_active',
    'warps': 'sm__warps_active.avg.pct_of_peak_sustained_active', 'regs': 'launch__registers_per_thread', 'smem': 'launch__shared_mem_per_block_dynamic',
    'l2_pct': 'lts__t_sectors.avg.pct_of_peak_sustained_elapsed', 'sm_pct': 'sm__throughput.avg.pct_of_peak_sustained_elapsed',
}
idx = {k: (hdr.index(v) if v in hdr else None) for k, v in want.items()}


def num(r, k):
    i = idx[k]
    if i is None or i >= len(r) or r[i] in ('', 'n/a'):
        return None
    try:
        return float(r[i].replace(',', ''))
    except ValueError:
        return None


def scale(v, unit, kind):
    if v is None:
        return None
    u = unit.lower()
    if kind == 'time':
        return v * {'ns': 1e-3, 'nsecond': 1e-3, 'us': 1.0, 'usecond': 1.0, 'ms': 1e3, 'msecond': 1e3, 's': 1e6, 'second': 1e6}.get(u, 1.0)
    return v * {'byte': 1.0, 'kbyte': 1e3, 'mbyte': 1e6, 'gbyte': 1e9}.get(u, 1.0)


print('%-58s %-14s %9s %10s %10s %7s %7s %7s %7s %5s' % ('kernel', 'grid', 'us', 'dram rd MB', 'dram wr MB', 'dram%', 'tensor%', 'L2%', 'warps%', 'regs'))
for r in rows[2:]:
    if len(r) < len(hdr):
        continue
    name = r[idx['name']].replace('void ', '').replace('<unnamed>::', '')[:58]
    dur = scale(num(r, 'dur'), units[idx['dur']] if idx['dur'] is not None else '', 'time')
    rd = scale(num(r, 'rd'), units[idx['rd']] if idx['rd'] is not None else '', 'bytes')
    wr = scale(num(r, 'wr'), units[idx['wr']] if idx['wr'] is not None else '', 'bytes')
    tp = num(r, 'tensor_pct')
    if tp is None:
        tp = num(r, 'tensor_pct2')
    f = lambda v, fmt: (fmt % v) if v is not None else '-'
    print('%-58s %-14s %9s %10s %10s %7s %7s %7s %7s %5s' % (name, r[idx['grid']].replace(' ', ''), f(dur, '%.1f'), f(rd / 1e6 if rd is not None else None, '%.2f'),
                                                          f(wr / 1e6 if wr is not None else None, '%.2f'), f(num(r, 'dram_pct'), '%.1f'), f(tp, '%.1f'),
                                                          f(num(r, 'l2_pct'), '%.1f'), f(num(r, 'warps'), '%.1f'), f(num(r, 'regs'), '%d')))
