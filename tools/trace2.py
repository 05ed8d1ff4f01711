"""Reads a SKYOPT_TRACE dump (skyopt_optimize_timed, last iteration): per
kernel (0 scan2, 1 place, 2 solve) and block 16 u64 slots of %globaltimer
marks. Prints, relative to the earliest mark, the spread of every mark.

    SKYOPT_TRACE=gpurun_out/trace.bin python bench.py ... ; python tools/trace2.py gpurun_out/trace.bin
"""
import sys

import numpy as np

KB, KS = 4096, 16
NAMES = {
    0: ['start', 'staged', 'tables', 'streamed', 'end'],
    # place: 'published' = minima and candidate count out (a chain block may
    # start), 'end' = candidate tables written
    1: ['start', 'resolved', 'counted', 'end', 'published'],
    # solve (chain DP): 'minima' = a chain block of its own saw every task's
    # minima, 'tables' = ... every task's tables (both absent when the chain
    # ran on the block that placed the DAG's last task)
    2: ['start', 'loaded', 'minima', 'recurrence', 'full-eval', 'backtrack',
        'end', 'tables'],
}


def main(path):
    a = np.fromfile(path, dtype=np.uint64).reshape(3, KB, KS)
    t0 = None
    for k in range(3):
        used = a[k][:, 0] > 0
        if used.any():
            m = a[k][used, 0].min()
            t0 = m if t0 is None else min(t0, m)
    for k, label in enumerate(['scan2', 'place', 'solve']):
        blk = a[k][a[k][:, 0] > 0]
        if not len(blk):
            continue
        print(f'{label}: {len(blk)} blocks')
        for i, name in enumerate(NAMES[k]):
            v = blk[:, i]
            v = v[v > 0].astype(np.float64) - float(t0)
            if len(v):
                print(f'  {name:10s} min {v.min()/1e3:7.2f}  p50 {np.median(v)/1e3:7.2f}'
                      f'  max {v.max()/1e3:7.2f} us')
        if k == 0:
            c = blk[:, 5]
            visit = (c & np.uint64(0xFFFFFFFF)).astype(np.int64)
            live = (c >> np.uint64(32)).astype(np.int64)
            print(f'  chunk visits {visit.sum()} live {live.sum()} '
                  f'(per block max {visit.max()})  SMs {len(set(blk[:, 6].tolist()))}')
            cyc = blk[:, 7].astype(np.float64)
            dur = (blk[:, 2].astype(np.float64) - blk[:, 1].astype(np.float64))
            ok = (cyc > 0) & (dur > 0)
            if ok.any():
                print(f'  table build: {np.median(cyc[ok]):.0f} cycles p50 in '
                      f'{np.median(dur[ok]):.0f} ns -> {np.median(cyc[ok] / dur[ok]):.2f} GHz')
        if k == 2:
            cyc = blk[:, 8].astype(np.float64)
            dur = blk[:, 3].astype(np.float64) - blk[:, 1].astype(np.float64)
            ok = (cyc > 0) & (dur > 0)
            if ok.any():
                print(f'  recurrence: {cyc[ok][0]:.0f} cycles in {dur[ok][0]:.0f} ns -> '
                      f'{cyc[ok][0] / dur[ok][0]:.2f} GHz')
            if blk.shape[1] > 12 and blk[0, 9:13].any():
                print('  one recurrence step (cycles): operands '
                      f'{int(blk[0, 9])}, sums + hazard {int(blk[0, 10])}, '
                      f'minimum {int(blk[0, 11])}, stores + next {int(blk[0, 12])}')


if __name__ == '__main__':
    main(sys.argv[1])
