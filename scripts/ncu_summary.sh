#!/usr/bin/env bash
# Text summary of an ncu report: launch header, the headline counters, the top source lines by stall samples.
#   scripts/ncu_summary.sh prof.ncu-rep > <kernel>_ncu_summary.txt
set -euo pipefail
rep="$1"
echo "# ncu summary of $(basename "$rep") (ncu --set full --clock-control none --import-source on; one launch)"
ncu -i "$rep" --page details 2>/dev/null | grep -E "^  [a-zA-Z_].*\(|Duration|Executed Ipc|Issue Slots Busy|Registers Per|Achieved Occupancy|Theoretical Occ|DRAM Throughput|Memory Throughput|L1/TEX Hit|L2 Hit Rate|No Eligible|Eligible Warps|Dynamic Shared Memory Per Block|Block Limit|Executed Instructions  |Grid Size|Waves Per SM" || true
echo "# raw counters"
ncu -i "$rep" --page raw --csv 2>/dev/null | python3 -c "
import csv, sys
r = list(csv.reader(sys.stdin)); h = r[0]
want = ['dram__bytes_read.sum', 'dram__bytes_write.sum', 'gpu__time_duration.sum', 'sm__warps_active.avg.pct_of_peak_sustained_active',
        'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active', 'sm__inst_executed.sum', 'launch__registers_per_thread',
        'dram__throughput.avg.pct_of_peak_sustained_elapsed', 'lts__t_sector_hit_rate.pct']
for row in r[2:]:
    name = row[h.index('Kernel Name')] if 'Kernel Name' in h else ''
    print(name[:60], {k: (row[h.index(k)], r[1][h.index(k)]) for k in want if k in h})
"
echo "# source lines by stall samples"
python3 "$(dirname "$0")/ncu_lines.py" "$rep" 25
