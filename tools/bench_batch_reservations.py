"""A controller's rounds when reserved capacity moves: the cfg5 workload
(10 000 single-task DAGs) on the reservation fixtures' catalog (6 000 rows,
AWS / GCP / Azure / Lambda), over twelve placement contexts with AWS and GCP
reservations enabled. After a first solve, every round changes two
contexts' inventories (new counts) and blocks the current placement of 10 %
of the DAGs (a region or zone wildcard on that DAG's own list).

Per-round wall time (p50 over the rounds, ms) of
  contexts_update   BatchOptimizerSession.optimize(lists, contexts=...): the
                    open session takes the new inventories on the device and
                    re-solves the forced and the re-priced DAGs
  fresh_session     a new batch_session per round (what a changed
                    process-wide inventory costs: a full statement and solve)
  optimize_batch    optimize_batch(dags, blocked_resources_per_dag=...,
                    contexts=...)
and the DAGs the first arm re-solved each round. Every arm's plans are
checked against the first arm's each round. The card's name and power limit
are printed with the numbers.

    python tools/bench_batch_reservations.py [n_dags] [rounds] [contexts]
"""
import json
import statistics
import sys
import time

sys.path.insert(0, '.')
import numpy as np  # noqa: E402
import skypilot_b200 as sky  # noqa: E402
from skypilot_b200 import _native, synth  # noqa: E402
from tools import bench_batch  # noqa: E402
from tools import bench_batch_failover  # noqa: E402

CATALOG = {'seed': 7, 'n_rows': 6000,
           'clouds': ['aws', 'gcp', 'azure', 'lambda']}
PRIO = {'aws': {'prioritize_reservations': True},
        'gcp': {'prioritize_reservations': True}}


def _inventory(store, k, rng=None):
    """Context k's records on real AWS / GCP types and zones of the
    catalog; `rng` draws new counts."""
    inv = []
    for name in ('aws', 'gcp'):
        table = store.cloud(name)
        types = list(table.inst_index)[2 * k:2 * k + 40]
        zones = list(table.zone_exact)
        for j, inst in enumerate(types):
            count = (1 + (j + k) % 4 if rng is None else
                     int(rng.integers(0, 5)))
            inv.append(dict(cloud=name, instance_type=inst,
                            zone=zones[(7 * j + k) % len(zones)],
                            name=f'r{k}-{j}', available=count))
    return inv


def _contexts(inventories):
    return [sky.PlacementContext(config=PRIO, reservations=inv)
            for inv in inventories]


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 10000
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    n_ctx = int(sys.argv[3]) if len(sys.argv) > 3 else 12
    if _native.device_count() < 1:
        raise SystemExit('no CUDA device: nothing to measure')
    store = sky.catalog.load_frames(synth.make_catalogs(**CATALOG))
    sky.check.set_enabled_clouds(sky.check.ALL_CATALOG_CLOUDS)
    store.handle(0)
    arms = ('contexts_update', 'fresh_session', 'optimize_batch')
    dags = {a: bench_batch.make_dags(n) for a in arms}
    rng = np.random.default_rng(5)
    inventories = [_inventory(store, k) for k in range(n_ctx)]
    ctxs = _contexts(inventories)
    contexts = [ctxs[i % n_ctx] for i in range(n)]
    lists = [[] for _ in range(n)]
    session = sky.Optimizer.batch_session(dags['contexts_update'],
                                          contexts=contexts)
    first = session.optimize(lists, return_exceptions=True, contexts=contexts)
    plans = [bench_batch_failover._record(o, d)  # pylint: disable=protected-access
             for o, d in zip(first, dags['contexts_update'])]
    times = {a: [] for a in arms}
    resolved, mismatches = [], 0
    for rnd in range(rounds):
        for k in rng.choice(n_ctx, size=2, replace=False):
            inventories[k] = _inventory(store, int(k), rng)
        ctxs = _contexts(inventories)
        contexts = [ctxs[i % n_ctx] for i in range(n)]
        live = [i for i, p in enumerate(plans) if not isinstance(p, str)]
        for i in rng.choice(live, size=n // 10, replace=False):
            lists[i] = lists[i] + [bench_batch_failover._wildcard(  # pylint: disable=protected-access
                plans[i], zone=bool((rnd + i) % 2))]
        got = {}
        t0 = time.perf_counter()
        out = session.optimize(lists, return_exceptions=True,
                               contexts=contexts)
        times['contexts_update'].append(1e3 * (time.perf_counter() - t0))
        resolved.append(sum(len(s.last_dag_ids or [])
                            for s in session._sessions if s is not None))  # pylint: disable=protected-access
        got['contexts_update'] = out
        t0 = time.perf_counter()
        with sky.Optimizer.batch_session(dags['fresh_session'],
                                         contexts=contexts) as fresh:
            got['fresh_session'] = fresh.optimize(lists,
                                                  return_exceptions=True)
        times['fresh_session'].append(1e3 * (time.perf_counter() - t0))
        t0 = time.perf_counter()
        got['optimize_batch'] = sky.optimize_batch(
            dags['optimize_batch'], blocked_resources_per_dag=lists,
            contexts=contexts, return_exceptions=True)
        times['optimize_batch'].append(1e3 * (time.perf_counter() - t0))
        recs = {a: [bench_batch_failover._record(o, d)  # pylint: disable=protected-access
                    for o, d in zip(got[a], dags[a])] for a in arms}
        plans = recs['contexts_update']
        for a in arms[1:]:
            mismatches += sum(x != y for x, y in zip(plans, recs[a]))
    session.close()
    result = dict(bench_batch_failover._card(), n_dags=n, contexts=n_ctx,  # pylint: disable=protected-access
                  rounds=rounds, mismatches=mismatches,
                  resolved_per_round=resolved,
                  errors=sum(isinstance(p, str) for p in plans))
    for arm, ts in times.items():
        result[f'{arm}_p50_ms'] = round(statistics.median(ts), 1)
        result[f'{arm}_ms'] = [round(t, 1) for t in ts]
    print(json.dumps(result))


if __name__ == '__main__':
    main()
