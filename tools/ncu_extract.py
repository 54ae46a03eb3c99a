"""Per-kernel table of the ncu metrics the profile notes quote, from an `ncu -i x.ncu-rep --page raw --csv` dump.

    python tools/ncu_extract.py raw.csv
"""
import csv
import sys

METRICS = [
    'gpu__time_duration.sum', 'dram__bytes_read.sum', 'dram__bytes_write.sum', 'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed',
    'sm__throughput.avg.pct_of_peak_sustained_elapsed', 'sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active',
    'sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active', 'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active',
    'sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active',
    'smsp__issue_active.avg.pct_of_peak_sustained_active', 'sm__warps_active.avg.pct_of_peak_sustained_active',
    'l1tex__m_xbar2l1tex_read_bytes.sum', 'lts__t_sector_hit_rate.pct', 'l1tex__data_pipe_lsu_wavefronts_mem_shared.sum',
    'l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum', 'launch__registers_per_thread', 'launch__shared_mem_per_block_dynamic',
    'launch__waves_per_multiprocessor', 'launch__grid_size', 'launch__block_size', 'smsp__inst_executed.sum',
]


def main(path):
    rows = list(csv.reader(open(path)))
    hdr = rows[0]
    units = rows[1]
    col = {h: i for i, h in enumerate(hdr)}
    kcol = col['Kernel Name']
    seen = {}
    for r in rows[2:]:
        seen.setdefault(r[kcol].split('(')[0], r)
    names = list(seen)
    print('| metric | unit | ' + ' | '.join(n.replace('glamr::', '').replace('void ', '') for n in names) + ' |')
    print('|---|---|' + '---|' * len(names))
    for m in METRICS:
        if m not in col:
            continue
        print(f'| {m} | {units[col[m]]} | ' + ' | '.join(seen[n][col[m]] for n in names) + ' |')


if __name__ == '__main__':
    main(sys.argv[1])
