"""`ncu --page raw --csv` export -> a short per-launch table (duration, DRAM bytes and GB/s, L2 -> SM bytes, L2 hit rate,
tensor-pipe / issue activity, registers, grid).  Usage: python tools/ncu_summary.py raw.csv [title] > summary.txt"""
import csv
import sys

COLS = [('gpu__time_duration.sum', 'us', 1.0),
        ('dram__bytes_read.sum', 'dram rd MB', 1.0),
        ('dram__bytes_write.sum', 'dram wr MB', 1.0),
        ('l1tex__m_xbar2l1tex_read_bytes.sum', 'L2->SM GB', 1.0),
        ('lts__t_sector_hit_rate.pct', 'L2 hit %', 1.0),
        ('sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active', 'tensor %', 1.0),
        ('smsp__issue_active.avg.pct_of_peak_sustained_active', 'issue %', 1.0),
        ('sm__warps_active.avg.pct_of_peak_sustained_active', 'occup %', 1.0),
        ('sm__cycles_active.avg', 'SM cycles', 1.0),
        ('launch__registers_per_thread', 'regs', 1.0),
        ('launch__grid_size', 'grid', 1.0)]


def main():
    rows = list(csv.reader(open(sys.argv[1])))
    hdr, units = rows[0], rows[1]
    idx = {h: i for i, h in enumerate(hdr)}
    if len(sys.argv) > 2:
        print(sys.argv[2])
    print('%-58s' % 'kernel' + ''.join('%12s' % c[1] for c in COLS) + '%12s' % 'DRAM GB/s')
    for r in rows[2:]:
        name = r[idx['Kernel Name']].replace('void <unnamed>::', '').replace('<unnamed>::', '')
        name = name.split('(')[0][:56]
        vals = []
        for key, _, _ in COLS:
            if key in idx:
                v, u = float(r[idx[key]].replace(',', '')), units[idx[key]]
                if u in ('Kbyte',):
                    v /= 1e3
                if u in ('byte',):
                    v /= 1e6
                if key.startswith('l1tex__m_xbar') and u == 'Mbyte':
                    v /= 1e3
                if u == 'ms':
                    v *= 1e3
                if u == 'ns':
                    v /= 1e3
                vals.append(v)
            else:
                vals.append(float('nan'))
        us, rd, wr = vals[0], vals[1], vals[2]
        print('%-58s' % name + ''.join('%12.1f' % v if abs(v) < 1e6 else '%12.3g' % v for v in vals) + '%12.0f' % ((rd + wr) / us * 1e3 if us else 0))


if __name__ == '__main__':
    main()
