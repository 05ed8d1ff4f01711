"""CPU model of the class-table scan's pruning, per block, for the piece plan
of equal chunk counts and for the cost-weighted plan (DESIGN §4).

For each piece it follows what a scan block does with the layout build_fast
makes: warp w takes chunks chunk_begin + w + 8 j; a chunk is scored when its
zone-map summary passes for some query of the group and its smallest rank
(`cmin`) is below that query's bound; scoring lowers each query's bound to
the chunk's smallest rank the query accepts. The block's warps share the
bound, modelled as one round of eight chunks at a time. It prints the
predicted live chunks and cost per block. With traces (SKYOPT_TRACE files of
the cfg4 fused step) it prints the measured counts beside them and fits the
cost constants: a block's time from `start` to `end` against its table-slice
entries, chunk visits and live chunks.

The plans come from the library (engine.scan_pieces), so the catalog is
built on a device; the model itself runs on the host.

    python tools/scan_model.py                       # predictions
    python tools/scan_model.py --record OUT          # + trace both plans to OUT/
    python tools/scan_model.py --traces EQ WEIGHTED  # + compare and fit
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from skypilot_b200 import _native, engine, workloads  # noqa: E402
from tests import scenario_runner as runner  # noqa: E402
from tests.test_gpu_chain_handoff import _state  # noqa: E402

ZR = _native.ZONE_ROWS
NONE = np.uint32(0xFFFFFFFF)
KB, KS = 4096, 16  # trace blocks, slots per block (skyopt_fast.cuh)


def ranks(cols, col):
    """Every row's rank in its cloud's (price, row) order (valid, priced
    rows; others NONE) for price column `col`."""
    price = cols['spot_price' if col else 'price']
    ok = ((cols['flags'] & _native.F_VALID) != 0) & ~np.isnan(price)
    out = np.full(len(price), NONE, np.uint32)
    offs = cols['cloud_row_offsets']
    for c in range(len(offs) - 1):
        r = np.arange(offs[c], offs[c + 1])
        r = r[ok[r]]
        order = r[np.lexsort((r, price[r]))]
        out[order] = np.arange(len(order), dtype=np.uint32)
    return out


def accepts(cols, sets, q, rows):
    """Rows of `rows` that query q accepts (the mask tables' rules)."""
    fl = cols['flags'][rows].astype(np.uint32)
    req = (int(q['flags_require']) | _native.F_VALID) & 0xFF
    ok = (fl & req) == req
    if q['group'] != 0:
        ok &= ((fl >> 8) & 0xFF) == (int(q['group']) & 0xFF)
    f2 = int(q['flags_require2'])
    ok &= (fl & f2) == f2
    if q['qflags'] & _native.Q_ACC:
        ak = cols['acc_key'][rows].astype(np.int64)
        words = sets[int(q['acc_set'])]
        has = ak != _native.NONE16
        bit = np.zeros(len(rows), bool)
        bit[has] = (words[ak[has] >> 5] >> (ak[has] & 31)) & 1 == 1
        ok &= bit
    if q['disk_op']:
        d = cols['disk_total'][rows]
        ok &= (d >= q['disk_size']) if q['disk_op'] == _native.DISK_GE else \
            (np.abs(d - q['disk_size']) < 1.0)
    v, m = cols['vcpus'][rows], cols['mem'][rows]
    with np.errstate(invalid='ignore'):
        if q['cpus_op']:
            hi = np.inf if q['cpus_op'] == _native.OP_GE else q['cpus']
            ok &= (v >= q['cpus']) & (v <= hi)
        if q['mem_op']:
            lo = v * q['mem'] if q['mem_op'] == _native.OP_RATIO else q['mem']
            hi = q['mem'] if q['mem_op'] == _native.OP_EQ else np.inf
            ok &= (m >= lo) & (m <= hi)
    if q['region_id'] >= 0:
        ok &= cols['region_id'][rows] == q['region_id']
    if q['zone_id'] >= 0:
        ok &= cols['zone_id'][rows] == q['zone_id']
    return ok


def zone_pass(zm, sets, q, chunks):
    req = (int(q['flags_require']) | _native.F_VALID) & 0xFF
    ok = (zm['flags_or'][chunks] & req) == req
    if q['group'] != 0:
        g = np.uint32(1 << (int(q['group']) & 31))
        ok &= (zm['groups'][chunks] & g) == g
    if q['qflags'] & _native.Q_ACC:
        s = sets[int(q['acc_set'])]
        lo, hi = np.bitwise_or.reduce(s[0::2]), np.bitwise_or.reduce(s[1::2])
        ok &= ((zm['sig_lo'][chunks] & lo) | (zm['sig_hi'][chunks] & hi)) != 0
    return ok


def model(store, queries, sets, plan, rank_cols, cmin_cols):
    """Per piece: (visits, predicted live chunks, slice entries, cloud)."""
    cols, zm = store.columns, store.columns['zone_map']
    out = []
    for p in plan.pieces:
        qs = queries[plan.group_queries[p['group']]]
        col = int(p['col'])
        chunks = np.arange(p['chunk_begin'], p['chunk_end'])
        n = len(chunks)
        rows = (chunks[:, None] * ZR + np.arange(ZR)).ravel()
        rk = rank_cols[col][rows].reshape(n, ZR)
        passes = np.stack([zone_pass(zm, sets, q, chunks) for q in qs])
        best = np.stack([np.where(accepts(cols, sets, q, rows).reshape(n, ZR),
                                  rk, NONE).min(axis=1) for q in qs])
        cmin = cmin_cols[col][chunks]
        bound = np.full(len(qs), NONE, np.uint32)
        live = 0
        for j in range(0, n, 8):  # one round: every warp's j-th chunk
            rnd = np.arange(j, min(j + 8, n))
            hit = passes[:, rnd] & (cmin[rnd][None, :] < bound[:, None])
            scored = rnd[hit.any(axis=0)]
            live += len(scored)
            if len(scored):
                bound = np.minimum(bound, best[:, scored].min(axis=1))
        out.append((n, live, int(p['slice_entries']), int(p['cloud'])))
    return np.array(out, dtype=np.int64).reshape(-1, 4)


def read_trace(path):
    a = np.fromfile(path, dtype=np.uint64).reshape(3, KB, KS)[0]
    used = a[:, 0] > 0
    blk = a[used]
    t0 = float(blk[:, 0].min())
    c = blk[:, 5]
    visits = (c & np.uint64(0xFFFFFFFF)).astype(np.int64)
    live = (c >> np.uint64(32)).astype(np.int64)
    return {'start': blk[:, 0].astype(np.float64) - t0,
            'tables': blk[:, 2].astype(np.float64) - t0,
            'end': blk[:, 4].astype(np.float64) - t0,
            'visits': visits, 'live': live}


def spread(x):
    return f'{x.min():.0f} / {np.median(x):.0f} / {x.max():.0f}'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='cfg4', choices=['cfg2', 'cfg4'])
    ap.add_argument('--record', metavar='DIR')
    ap.add_argument('--traces', nargs=2, metavar=('EQUAL', 'WEIGHTED'))
    ap.add_argument('--cost', nargs=3, type=float, default=(5.0, 23.0, 68.0),
                    metavar=('C_E', 'C_V', 'C_L'),
                    help='ns per table entry, chunk visit and live chunk '
                    '(kCostEntry, kCostVisit, kCostLive in skyopt.cu)')
    args = ap.parse_args()
    store = runner.activate_catalog(workloads.CATALOGS[args.workload])
    dag, _ = workloads.build_dag(
        workloads.chain_scenario(32 if args.workload == 'cfg4' else 8))
    builder = engine.ProblemBuilder(store)
    _state(dag, builder)
    packed = builder.pack()
    queries = packed.queries[:packed.n_queries]
    sets = engine.set_table(store).reshape(-1, _native.ACC_SET_WORDS)
    cols = store.columns
    rank_cols = [ranks(cols, 0), ranks(cols, 1)]
    cmin_cols = [r.reshape(-1, ZR).min(axis=1) for r in rank_cols]
    names = {i: t.name for i, t in enumerate(store.clouds)}
    traces = list(args.traces) if args.traces else None
    if args.record:
        os.makedirs(args.record, exist_ok=True)
        # the library names the n-th timing loop's trace <path>.<n> (n > 0)
        path = os.path.join(args.record, 'trace.bin')
        traces = [path, path + '.1']
        os.environ['SKYOPT_TRACE'] = path
        try:
            for equal in (True, False):
                engine.set_scan_pieces(equal=equal)
                engine.solve_timed(builder, 5, True)
        finally:
            engine.set_scan_pieces()
            del os.environ['SKYOPT_TRACE']
    fit_rows = []
    for k, (label, equal) in enumerate((('equal', True), ('weighted', False))):
        engine.set_scan_pieces(equal=equal)
        try:
            plan = engine.scan_pieces(builder, fused=True)
        finally:
            engine.set_scan_pieces()
        m = model(store, queries, sets, plan, rank_cols, cmin_cols)
        print(f'== {label} pieces: {len(m)} blocks (grid {plan.grid})')
        print(f'  predicted live chunks per block min / p50 / max: '
              f'{spread(m[:, 1])}  ({m[:, 1].sum()} in all)')
        ce, cv, cl = args.cost
        cost = m[:, 2] * ce + m[:, 0] * cv + m[:, 1] * cl
        print(f'  predicted cost per block (ns) min / p50 / max: {spread(cost)}')
        for c in np.unique(m[:, 3]):
            sel = m[:, 3] == c
            print(f'    {names[int(c)]:8s} pieces {sel.sum():4d}  chunks '
                  f'{m[sel, 0].sum():6d}  live {m[sel, 1].sum():5d}  '
                  f'max per piece {m[sel, 1].max():3d}')
        if traces:
            t = read_trace(traces[k])
            n = min(len(m), len(t['live']))
            print(f'  measured live per block min / p50 / max: '
                  f'{spread(t["live"][:n])}  ({t["live"][:n].sum()} in all); '
                  f'visits match the plan: '
                  f'{bool((t["visits"][:n] == m[:n, 0]).all())}')
            print(f'  marks (ns) tables {spread(t["tables"])}  '
                  f'end {spread(t["end"])}')
            fit_rows.append(np.column_stack([
                np.ones(n), m[:n, 2], t['visits'][:n], t['live'][:n],
                t['end'][:n] - t['start'][:n]]))
    if fit_rows:
        x = np.vstack(fit_rows)
        coef, *_ = np.linalg.lstsq(x[:, :4], x[:, 4], rcond=None)
        print(f'fit of block time (ns) over both traces, {len(x)} blocks: '
              f'{coef[0]:.0f} + {coef[1]:.2f} per entry + {coef[2]:.2f} per '
              f'visit + {coef[3]:.1f} per live chunk')


if __name__ == '__main__':
    main()
