"""profiles/conv_traffic.json from an ncu launch list (tools/gpu_launchlist.sh): DRAM bytes of the conv kernels of
ONE training step, stamped with the hash of the kernel sources they were measured with (bench.py refuses a stale file).
usage: python tools/conv_traffic_from_launchlist.py launchlist_out/launches_resnet50.csv resnet50_uq8_dst_b128 128"""
import csv
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402


def main():
    path, workload, batch = sys.argv[1], sys.argv[2], int(sys.argv[3])
    lines = [l for l in open(path) if l.startswith('"')]
    rows, cur = [], {}
    for r in csv.DictReader(lines):
        k = r['ID']
        if k not in cur:
            cur[k] = dict(name=r['Kernel Name'])
            rows.append(cur[k])
        v = float(r['Metric Value'].replace(',', '')) if r['Metric Value'] not in ('', 'n/a') else 0.0
        scale = dict(byte=1, Kbyte=1e3, Mbyte=1e6, Gbyte=1e9).get(r['Metric Unit'], 1)
        if r['Metric Name'].startswith('dram__bytes'):
            cur[k][r['Metric Name']] = v * scale
    marks = [i for i, r in enumerate(rows) if 'softmax_ce_rows' in r['name']]
    if len(marks) >= 2:
        rows = rows[marks[0]:marks[1]]
    conv = [r for r in rows if any(t in r['name'] for t in ('conv_tma', 'conv_tc_', 'tc_prep', 'tc_splitk', 's2d_planes'))]
    total = sum(r.get('dram__bytes_read.sum', 0.0) + r.get('dram__bytes_write.sum', 0.0) for r in conv)
    out = dict(workload=workload, batch=batch, conv_dram_bytes_per_step=total, conv_launches=len(conv),
               kernel_source_stamp=bench.kernel_source_stamp(), source=os.path.basename(path))
    os.makedirs(os.path.join(bench.ROOT, 'profiles'), exist_ok=True)
    json.dump(out, open(os.path.join(bench.ROOT, 'profiles', 'conv_traffic.json'), 'w'), indent=1)
    print(out)


if __name__ == '__main__':
    main()
