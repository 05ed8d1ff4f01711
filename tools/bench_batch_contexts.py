"""Launches of several workspaces planned together: the cfg5 workload (10 000
single-task DAGs on the 50 000-row catalog) spread over eight placement
contexts -- different enabled clouds, SkyPilot configs, reservation
inventories and objectives.

Wall time per pass (p50 over the repetitions, ms) of
  one_call      optimize_batch(dags, contexts=...): one device problem
  per_context   one optimize_batch per context, the process state set to
                that context before each call (what a controller had to do
                before contexts)
The two arms' plans are checked against each other on every repetition.
The card's name and power limit are printed with the numbers.

    python tools/bench_batch_contexts.py [n_dags] [repetitions]
"""
import json
import statistics
import sys
import time

sys.path.insert(0, '.')
import skypilot_b200 as sky  # noqa: E402
from skypilot_b200 import _native, synth  # noqa: E402
from skypilot_b200 import check, reservations, skypilot_config  # noqa: E402
from tools import bench_batch  # noqa: E402
from tools import bench_batch_failover  # noqa: E402


def _contexts(store):
    """Eight workspaces: cloud subsets, reservation configs and inventories
    on real AWS / GCP types of the catalog, COST and TIME."""
    clouds = [t.name for t in store.clouds]
    out = []
    for k in range(8):
        inv = []
        for name in ('aws', 'gcp'):
            table = store.cloud(name)
            types = list(table.inst_index)[k:k + 24]
            zones = list(table.zone_exact)
            for j, inst in enumerate(types):
                inv.append(dict(cloud=name, instance_type=inst,
                                zone=zones[(7 * j + k) % len(zones)],
                                name=f'r{k}-{j}', available=1 + (j + k) % 4))
        prio = {c: {'prioritize_reservations': True}
                for c in (('aws',), ('gcp',), ('aws', 'gcp'))[k % 3]}
        out.append(sky.PlacementContext(
            enabled_clouds=clouds[:2 + k % 3] if k % 4 else None,
            config=prio if k % 2 == 0 else {},
            reservations=inv,
            minimize=(sky.OptimizeTarget.TIME if k % 4 == 3 else
                      sky.OptimizeTarget.COST)))
    return out


def _record(o, dag):
    if isinstance(o, Exception):
        return str(o)
    r = dag.tasks[0].best_resources
    return (str(r.cloud), r.instance_type, r.region, r.zone)


def _per_context(dags, contexts):
    """One optimize_batch per context under that context's process state."""
    out = [None] * len(dags)
    groups = {}
    for i, ctx in enumerate(contexts):
        groups.setdefault(id(ctx), (ctx, []))[1].append(i)
    saved = (check._enabled, skypilot_config._config, reservations._records)  # pylint: disable=protected-access
    try:
        for ctx, idx in groups.values():
            check.set_enabled_clouds(
                list(ctx.enabled_clouds) if ctx.enabled_clouds is not None
                else check.ALL_CATALOG_CLOUDS)
            skypilot_config.set_config(ctx.config)
            reservations.set_reservations(ctx.reservations)
            got = sky.optimize_batch([dags[i] for i in idx], ctx.minimize,
                                     return_exceptions=True)
            for i, o in zip(idx, got):
                out[i] = o
    finally:
        check._enabled = saved[0]  # pylint: disable=protected-access
        skypilot_config.set_config(saved[1])
        reservations._records = saved[2]  # pylint: disable=protected-access
    return out


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 10000
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    if _native.device_count() < 1:
        raise SystemExit('no CUDA device: nothing to measure')
    store = sky.catalog.load_frames(synth.make_catalogs(1, 50000))
    check.set_enabled_clouds(check.ALL_CATALOG_CLOUDS)
    store.handle(0)
    ctxs = _contexts(store)
    contexts = [ctxs[i % len(ctxs)] for i in range(n)]
    dags = {'one_call': bench_batch.make_dags(n),
            'per_context': bench_batch.make_dags(n)}
    arms = {
        'one_call': lambda: sky.optimize_batch(
            dags['one_call'], contexts=contexts, return_exceptions=True),
        'per_context': lambda: _per_context(dags['per_context'], contexts),
    }
    times = {a: [] for a in arms}
    mismatches = 0
    for rep in range(reps + 1):  # the first pass warms up both arms
        plans = {}
        for arm, fn in arms.items():
            t0 = time.perf_counter()
            out = fn()
            ms = 1e3 * (time.perf_counter() - t0)
            if rep:
                times[arm].append(ms)
            plans[arm] = [_record(o, d) for o, d in zip(out, dags[arm])]
        mismatches += sum(a != b for a, b in zip(plans['one_call'],
                                                 plans['per_context']))
    result = dict(bench_batch_failover._card(), n_dags=n, contexts=len(ctxs),  # pylint: disable=protected-access
                  repetitions=reps, mismatches=mismatches,
                  errors=sum(isinstance(p, str) for p in plans['one_call']))
    for arm, ts in times.items():
        result[f'{arm}_p50_ms'] = round(statistics.median(ts), 1)
        result[f'{arm}_ms'] = [round(t, 1) for t in ts]
    print(json.dumps(result))


if __name__ == '__main__':
    main()
