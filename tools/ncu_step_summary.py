"""Condenses `ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --csv` of ONE eager training step
(bench.py brackets its instrumented step with cudaProfilerStart / Stop) into a per-kernel table and the DRAM-traffic JSON bench.py reads for `roofline.traffic`.

    ncu --profile-from-start off --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum \\
        --clock-control none --csv --log-file tools_out/launches.csv python bench.py --steps 1 --warmup 3 --graph 0 --no-cpu-baseline
    python tools/ncu_step_summary.py tools_out/launches.csv tools_out/ncu_launch_summary.txt tools_out/ncu_traffic.json
"""
import collections
import csv
import json
import sys


def main(src, out_txt, out_json):
    rows = [r for r in csv.reader(l for l in open(src) if l.startswith('"'))]
    h = rows[0]
    ki, mi, vi, ui = h.index('Kernel Name'), h.index('Metric Name'), h.index('Metric Value'), h.index('Metric Unit')
    agg = collections.defaultdict(lambda: [0, 0.0, 0.0])
    for r in rows[1:]:
        v = float(r[vi].replace(',', ''))
        k = r[ki].replace('void ', '').replace('<unnamed>::', '').split('(')[0][:60]
        if r[mi] == 'gpu__time_duration.sum':
            agg[k][0] += 1
            agg[k][1] += v / 1e3 if r[ui] in ('ns', 'nsecond') else v
        else:
            agg[k][2] += v * {'byte': 1, 'Kbyte': 1e3, 'Mbyte': 1e6, 'Gbyte': 1e9}.get(r[ui], 1)
    tot = sum(v[1] for v in agg.values())
    with open(out_txt, 'w') as f:
        f.write('one eager training step (batch 10, bf16 mode) under ncu --metrics gpu__time_duration.sum,dram__bytes_* (serialised, cold caches; '
                'cudaProfilerStart/Stop around the step): %d launches, %.2f ms of kernel time\n' % (sum(v[0] for v in agg.values()), tot / 1e3))
        for k, (n, us, by) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            f.write('%9.1f us %5.1f%% x%-5d %9.2f MB DRAM/launch  %s\n' % (us, 100 * us / tot, n, by / max(n, 1) / 1e6, k))
    g = [(k, v) for k, v in agg.items() if 'gemm_tc_kernel' in k]
    n = sum(v[0] for _, v in g)
    by = sum(v[2] for _, v in g)
    json.dump({'gemm_tc_kernel': {'dram_bytes_per_launch': round(by / max(n, 1)), 'launches': n,
                                  'source': 'ncu dram__bytes_read.sum + dram__bytes_write.sum over the %d gemm_tc_kernel launches of one eager step (%s)'
                                            % (n, out_txt)}}, open(out_json, 'w'))
    print(open(out_txt).read()[:3000])


if __name__ == '__main__':
    main(*sys.argv[1:4])
