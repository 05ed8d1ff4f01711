"""Failover of many launches at once on the cfg5 workload: 10 000 single-task
DAGs on the 50 000-row catalog, 5 rounds after a first full solve, each round
blocking the current placement of 10 % of the DAGs (a region or zone
wildcard added to that DAG's own list).

Per-round wall time (p50 over the rounds, ms) of
  resolve_dags_changed   BatchOptimizerSession.optimize: only the DAGs whose
                         list changed are filtered, solved and read back
  resolve_dags_all       the same, with every DAG listed to the device
  optimize_batch         optimize_batch(dags, blocked_resources_per_dag=...)
  per_dag_sessions       one OptimizerSession per DAG, the changed ones
                         called; measured on a sample and scaled to all DAGs
Every arm's plans are checked against the first arm's each round. The card's
name and power limit are printed with the numbers.

    python tools/bench_batch_failover.py [n_dags] [rounds] [session_sample]
"""
import json
import statistics
import subprocess
import sys
import time

sys.path.insert(0, '.')
import numpy as np  # noqa: E402
import skypilot_b200 as sky  # noqa: E402
from skypilot_b200 import _native, synth  # noqa: E402
from skypilot_b200 import optimizer as opt_lib  # noqa: E402
from skypilot_b200.utils import registry  # noqa: E402
from tools import bench_batch  # noqa: E402


class _AllListed(opt_lib.BatchOptimizerSession):
    """Lists every DAG to the device on each re-solve (reads back the
    changed ones only, like the session it is compared with)."""

    def _resolve(self, todo, packed):
        super()._resolve(list(range(len(self.dags))), packed)


def _card():
    try:
        line = subprocess.run(
            ['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
             '--format=csv,noheader', '-i', '0'], capture_output=True,
            text=True, timeout=60, check=True).stdout.strip()
        name, power, sm = [x.strip() for x in line.split(',')]
        return {'gpu': name, 'power_limit': power, 'sm_clock_max': sm}
    except (OSError, subprocess.SubprocessError, ValueError):
        return {'gpu': 'unknown', 'power_limit': 'unknown'}


def _record(o, dag):
    if isinstance(o, Exception):
        return str(o)
    r = dag.tasks[0].best_resources
    return (str(r.cloud), r.instance_type, r.region, r.zone)


def _wildcard(rec, zone):
    cloud, inst, region, z = rec
    kw = dict(cloud=registry.CLOUD_REGISTRY.from_str(cloud), region=region)
    if zone and z is not None:
        kw['zone'] = z
    r = sky.Resources(**kw)
    r._use_spot_specified = False  # pylint: disable=protected-access
    return r


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 10000
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    sample = int(sys.argv[3]) if len(sys.argv) > 3 else 500
    if _native.device_count() < 1:
        raise SystemExit('no CUDA device: nothing to measure')
    frames = synth.make_catalogs(1, 50000)
    store = sky.catalog.load_frames(frames)
    sky.check.set_enabled_clouds(sky.check.ALL_CATALOG_CLOUDS)
    store.handle(0)
    arms = ('resolve_dags_changed', 'resolve_dags_all', 'optimize_batch',
            'per_dag_sessions')
    dags = {a: bench_batch.make_dags(n) for a in arms[:3]}
    dags['per_dag_sessions'] = bench_batch.make_dags(n)[:sample]
    sky.optimize_batch(bench_batch.make_dags(200), return_exceptions=True)
    rng = np.random.default_rng(5)
    lists = [[] for _ in range(n)]
    changed = opt_lib.BatchOptimizerSession(dags['resolve_dags_changed'])
    every = _AllListed(dags['resolve_dags_all'])
    singles = [sky.Optimizer.session(d) for d in dags['per_dag_sessions']]
    times = {a: [] for a in arms}

    def timed(arm, fn):
        t0 = time.perf_counter()
        out = fn()
        times[arm].append(1e3 * (time.perf_counter() - t0))
        return out

    mismatches = 0
    touched = list(range(n))
    for rnd in range(rounds + 1):
        out = timed(arms[0], lambda: changed.optimize(lists,
                                                      return_exceptions=True))
        want = [_record(o, d) for o, d in zip(out, dags[arms[0]])]
        out = timed(arms[1], lambda: every.optimize(lists,
                                                    return_exceptions=True))
        mismatches += sum(_record(o, d) != w for o, d, w in
                          zip(out, dags[arms[1]], want))
        out = timed(arms[2], lambda: sky.optimize_batch(
            dags[arms[2]], blocked_resources_per_dag=lists,
            return_exceptions=True))
        mismatches += sum(_record(o, d) != w for o, d, w in
                          zip(out, dags[arms[2]], want))

        def per_dag():
            for i in touched:
                if i >= sample:
                    break
                try:
                    singles[i].optimize(lists[i])
                except sky.exceptions.ResourcesUnavailableError:
                    pass

        timed(arms[3], per_dag)
        # the next round's failed launches: 10 % of the DAGs with a plan
        live = [i for i, w in enumerate(want) if isinstance(w, tuple)]
        touched = sorted(int(i) for i in rng.choice(
            live, size=min(len(live), n // 10), replace=False))
        for i in touched:
            lists[i].append(_wildcard(want[i], zone=(rnd + i) % 2 == 0))
    changed.close()
    every.close()
    for s in singles:
        s.close()
    result = {
        'workload': (f'cfg5 failover: {n} single-task DAGs, '
                     f'{synth.total_rows(frames)}-row catalog, {rounds} '
                     f'rounds blocking {n // 10} DAGs each'),
        **_card(),
        'first_solve_ms': {a: round(times[a][0], 2) for a in arms[:3]},
        'p50_round_ms': {a: round(statistics.median(times[a][1:]), 2)
                         for a in arms[:3]},
        'per_dag_sessions_p50_round_ms_scaled': round(
            statistics.median(times[arms[3]][1:]) * n / sample, 2),
        'per_dag_sessions_sample': sample,
        'round_ms': {a: [round(t, 2) for t in times[a]] for a in arms},
        'plan_mismatches': mismatches,
    }
    print(json.dumps(result))


if __name__ == '__main__':
    main()
