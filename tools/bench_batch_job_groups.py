"""A controller's queue with JobGroups: seeded JobGroups of 1-8 jobs mixed
with cfg5-style single-task DAGs (one single-task DAG per group) on the
multi50k catalog (50 000 rows, AWS / GCP / Azure / Lambda).

Wall time (p50, ms) of
  batch             optimize_batch(dags, job_groups=True): every group and
                    DAG in one device problem
  loop              optimize_job_group per group and optimize_batch for the
                    single-task DAGs (what a controller did before)
  session_round     BatchOptimizerSession(job_groups=True) rounds, each
                    blocking the chosen region of 10 % of the groups
  single_device     one optimize_job_group call (a 4-job group)
  single_host       the same group through the host algorithm that
                    optimize_job_group ran before (_optimize_job_group_host:
                    candidate tables copied back, selection in Python),
                    alternated with single_device in this process
Plans of `batch` and `loop` are compared every repetition, and every
session round against a fresh optimize_batch. The card's name and power
limit are printed with the numbers.

    python tools/bench_batch_job_groups.py [n_groups] [reps] [rounds]
"""
import json
import random
import statistics
import sys
import time

sys.path.insert(0, '.')
import skypilot_b200 as sky  # noqa: E402
from skypilot_b200 import _native, synth  # noqa: E402
from skypilot_b200 import optimizer as opt_lib  # noqa: E402
from skypilot_b200.dag import DagExecution  # noqa: E402
from skypilot_b200.utils import registry  # noqa: E402
from tools import bench_batch  # noqa: E402
from tools import bench_batch_failover  # noqa: E402

CATALOG = {'seed': 1, 'n_rows': 50000,
           'clouds': ['aws', 'gcp', 'azure', 'lambda']}
_ACCS = [None, 'V100', 'T4', 'A100', 'A100:8', 'L4', 'K80', 'V100:4']


def make_groups(store, n, seed=9):
    """n JobGroups of 1-8 jobs: a third pinned to one cloud, a sixth to one
    region, some spot jobs and multi-node jobs."""
    rng = random.Random(seed)
    groups = []
    for k in range(n):
        shape = rng.random()
        table = rng.choice(store.clouds)
        region = rng.choice(table.region_names)
        with sky.Dag() as dag:
            for j in range(rng.randint(1, 8)):
                spec = {}
                acc = rng.choice(_ACCS)
                if acc:
                    spec['accelerators'] = acc
                else:
                    spec['cpus'] = rng.choice(['4+', '8+', '32+'])
                if shape < 0.5:
                    spec['cloud'] = registry.CLOUD_REGISTRY.from_str(
                        table.name)
                if shape < 0.17:
                    spec['region'] = region
                if rng.random() < 0.2:
                    spec['use_spot'] = True
                sky.Task(f'g{k}j{j}', num_nodes=rng.choice(
                    [1, 1, 1, 2, 4])).set_resources(sky.Resources(**spec))
        dag.name = f'g{k}'
        dag.set_execution(DagExecution.PARALLEL)
        groups.append(dag)
    return groups


def _record(o, dag):
    if isinstance(o, Exception):
        return str(o)
    return [(str(t.best_resources.cloud), t.best_resources.instance_type,
             t.best_resources.region, t.best_resources.zone)
            for t in dag.tasks]


def _block(rec):
    cloud, _, region, _ = rec[0]
    r = sky.Resources(cloud=registry.CLOUD_REGISTRY.from_str(cloud),
                      region=region)
    r._use_spot_specified = False  # pylint: disable=protected-access
    return r


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 2000
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    rounds = int(sys.argv[3]) if len(sys.argv) > 3 else 5
    if _native.device_count() < 1:
        raise SystemExit('no CUDA device: nothing to measure')
    store = sky.catalog.load_frames(synth.make_catalogs(**CATALOG))
    sky.check.set_enabled_clouds(sky.check.ALL_CATALOG_CLOUDS)
    store.handle(0)
    times = {'batch': [], 'loop': []}
    mismatches = 0
    for rep in range(reps + 1):  # the first repetition warms up
        dags = make_groups(store, n) + bench_batch.make_dags(n)
        t0 = time.perf_counter()
        out = sky.optimize_batch(dags, return_exceptions=True,
                                 job_groups=True)
        t_batch = 1e3 * (time.perf_counter() - t0)
        got = [_record(o, d) for o, d in zip(out, dags)]
        dags = make_groups(store, n) + bench_batch.make_dags(n)
        t0 = time.perf_counter()
        loop = []
        for dag in dags[:n]:
            try:
                loop.append(sky.Optimizer.optimize_job_group(dag, quiet=True))
            except sky.exceptions.ResourcesUnavailableError as e:
                loop.append(e)
        loop += sky.optimize_batch(dags[n:], return_exceptions=True)
        t_loop = 1e3 * (time.perf_counter() - t0)
        mismatches += sum(
            a != b for a, b in zip(got, [_record(o, d)
                                         for o, d in zip(loop, dags)]))
        if rep:
            times['batch'].append(t_batch)
            times['loop'].append(t_loop)
    # failover rounds of the groups
    groups = make_groups(store, n)
    lists = [[] for _ in groups]
    rng = random.Random(3)
    session_ms, resolved = [], []
    with sky.Optimizer.batch_session(groups, job_groups=True) as session:
        out = session.optimize(lists, return_exceptions=True)
        for _ in range(rounds):
            live = [i for i, o in enumerate(out)
                    if not isinstance(o, Exception)]
            for i in rng.sample(live, max(1, len(live) // 10)):
                lists[i] = lists[i] + [_block(_record(out[i], groups[i]))]
            t0 = time.perf_counter()
            out = session.optimize(lists, return_exceptions=True)
            session_ms.append(1e3 * (time.perf_counter() - t0))
            resolved.append(sum(len(s.last_dag_ids or [])
                                for s in session._sessions if s is not None))  # pylint: disable=protected-access
            fresh = make_groups(store, n)
            want = sky.optimize_batch(fresh, blocked_resources_per_dag=lists,
                                      return_exceptions=True, job_groups=True)
            mismatches += sum(
                _record(a, d) != _record(b, f)
                for a, b, d, f in zip(out, want, groups, fresh))
    # one group, the device path and the host algorithm alternated
    group = [g for g in make_groups(store, 200, seed=21)
             if len(g.tasks) == 4][0]
    opened = [(t, t.resources) for t in group.tasks]
    single = {'single_device': [], 'single_host': []}
    for k in range(2 * 41):
        arm = ('single_device', 'single_host')[k % 2]
        for t, resources in opened:  # undo the previous call's override
            t.resources = resources
        t0 = time.perf_counter()
        if arm == 'single_device':
            sky.Optimizer.optimize_job_group(group, quiet=True)
        else:
            opt_lib.Optimizer._optimize_job_group_host(  # pylint: disable=protected-access
                group, sky.OptimizeTarget.COST, [], quiet=True)
        if k >= 2:
            single[arm].append(1e3 * (time.perf_counter() - t0))
    result = dict(bench_batch_failover._card(), n_groups=n,  # pylint: disable=protected-access
                  n_single_task_dags=n, reps=reps, rounds=rounds,
                  mismatches=mismatches, resolved_per_round=resolved)
    for arm, ts in list(times.items()) + [('session_round', session_ms)] + list(
            single.items()):
        result[f'{arm}_p50_ms'] = round(statistics.median(ts), 3)
    result['batch_ms'] = [round(t, 1) for t in times['batch']]
    result['loop_ms'] = [round(t, 1) for t in times['loop']]
    result['session_round_ms'] = [round(t, 1) for t in session_ms]
    print(json.dumps(result))


if __name__ == '__main__':
    main()
