"""skyopt_solve_tables (solve_kernel) against the exact table-level model of
oracle/table_dp.py on the seeded regimes of tests/table_cases.py:

* chains of 1-32 tasks (the fused step's chain DP: the lean recurrence for at
  most four clouds, the general one's shuffle loop up to eight and butterfly
  beyond, the full evaluation after a hazard) and of 33-300 tasks (the
  per-candidate DP), on 1-22 clouds, under every chain knob: the same index
  per task and the same objective bits;
* a task without candidates first, in the middle or last;
* general DAGs of 2-16 tasks, COST and TIME: the exact optimum;
* the enumeration's limits (2^26 assignments, 16 tasks) and what
  _optimize_by_ilp does beyond them;
* several DAGs of different kinds in one launch.
The SKYOPT_EXP knobs are read once per process, hence the subprocesses."""
import json
import math
import os
import subprocess
import sys
from collections import Counter

import networkx as nx
import numpy as np
import pytest

from oracle import table_dp
from tests import table_cases

pytestmark = pytest.mark.gpu

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLOUD_COUNTS = (1, 2, 3, 4, 6, 9, 16, 22)
SHORT = (1, 2, 3, 8, 31, 32)
LONG = (33, 64, 300)


# ---- worker side (runs in a subprocess with the knob set) -------------------
def _store(n_clouds):
    from skypilot_b200 import synth  # pylint: disable=import-outside-toplevel
    from skypilot_b200.catalog.store import CatalogStore  # pylint: disable=import-outside-toplevel
    names = list(synth._MAKERS)[:n_clouds]  # pylint: disable=protected-access
    assert len(names) == n_clouds
    return CatalogStore.from_frames(
        synth.make_catalogs(seed=5, n_rows=40 * n_clouds, clouds=names))


def _device(store, tb, is_chain=True, minimize_cost=True):
    from skypilot_b200 import engine  # pylint: disable=import-outside-toplevel
    return engine.solve_tables(store, *tb.args(), is_chain, minimize_cost)


def _chain_check(store, tb):
    chosen, obj, status = _device(store, tb)
    empty = tb.first_empty()
    if empty is not None:
        ok = status == 1 and chosen == [-1] * tb.n_tasks
        return ok, f'status {status} chosen {chosen[:4]}'
    plan, want = table_dp.chain_dp(tb)
    ok = status == 0 and chosen == plan and obj.hex() == want.hex()
    return ok, f'status {status} obj {obj.hex()} want {want.hex()}'


def _chains(knob):
    """Every chain case on every cloud count; returns counts and failures."""
    counts, bad = Counter(), []
    for n_clouds in CLOUD_COUNTS:
        store = _store(n_clouds)
        for regime in table_cases.CHAIN_REGIMES:
            for n_tasks in SHORT + LONG:
                seeds = 2 if n_tasks in SHORT else 1
                for seed in range(seeds):
                    rng = np.random.default_rng([n_clouds, n_tasks, seed,
                                                 table_cases.CHAIN_REGIMES.index(regime)])
                    tb = table_cases.chain(rng, regime, n_tasks, n_clouds)
                    ok, why = _chain_check(store, tb)
                    path = 'short' if n_tasks in SHORT else 'long'
                    counts[f'{path}/{n_clouds}/{regime}/{knob}'] += 1
                    if not ok:
                        bad.append((regime, n_clouds, n_tasks, seed, why))
        if n_clouds > 1:
            for i, tb in enumerate(table_cases.signed_zero_chains(n_clouds)):
                ok, why = _chain_check(store, tb)
                counts[f'signed0/{n_clouds}/signed/{knob}'] += 1
                if not ok:
                    bad.append(('signed0', n_clouds, tb.n_tasks, i, why))
        # a task of 10^5 candidates, in a short and a long chain
        for n_tasks in (8, 40):
            rng = np.random.default_rng([n_clouds, n_tasks, 99])
            tb = table_cases.chain(rng, 'quantized', n_tasks, n_clouds,
                                   big_task=n_tasks // 2)
            ok, why = _chain_check(store, tb)
            counts[f'big/{n_clouds}/quantized/{knob}'] += 1
            if not ok:
                bad.append(('big', n_clouds, n_tasks, 0, why))
        # a task without candidates: first, middle, last
        for n_tasks in (1, 3, 8, 32, 40):
            for at in sorted({0, n_tasks // 2, n_tasks - 1}):
                rng = np.random.default_rng([n_clouds, n_tasks, at, 7])
                tb = table_cases.chain(rng, 'random', n_tasks, n_clouds,
                                       empty_at=at)
                if at + 1 < n_tasks:
                    tb.values[-1] = np.zeros(0)   # a later empty one too
                    tb.clouds[-1] = np.zeros(0, dtype=np.int64)
                ok, why = _chain_check(store, tb)
                counts[f'empty/{n_clouds}/random/{knob}'] += 1
                if not ok:
                    bad.append(('empty', n_clouds, n_tasks, at, why))
    return counts, bad


def main(knob):
    counts, bad = _chains(knob)
    print(json.dumps({'counts': counts, 'bad': bad[:20], 'n_bad': len(bad)}))


# ---- test side -------------------------------------------------------------
def _run(code, knob):
    env = dict(os.environ)
    env.pop('SKYOPT_EXP', None)
    if knob:
        env['SKYOPT_EXP'] = knob
    proc = subprocess.run([sys.executable, '-c', code], cwd=_ROOT, env=env,
                          capture_output=True, text=True, timeout=1200,
                          check=False)
    assert proc.returncode == 0, proc.stdout[-2000:] + proc.stderr[-2000:]
    return json.loads(proc.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize('knob', [None, '8', '16', '24'])
def test_chains_match_the_model(knob):
    """Unset: the default paths; 8: the full evaluation on every chain; 16:
    the general recurrence for every cloud count; 24: both."""
    out = _run('import sys; sys.path.insert(0, "."); '
               'from tests.test_gpu_dp_tables import main; '
               f'main({knob!r})', knob)
    print(json.dumps(out['counts'], sort_keys=True))
    assert out['n_bad'] == 0, out['bad']
    n = sum(out['counts'].values())
    assert n == len(CLOUD_COUNTS) * (
        len(table_cases.CHAIN_REGIMES) * (2 * len(SHORT) + len(LONG)) + 2 +
        sum(len({0, k // 2, k - 1}) for k in (1, 3, 8, 32, 40))) + 3 * (
            len(CLOUD_COUNTS) - 1)


# ---- general DAGs (no knob) ------------------------------------------------
def _options(rng, n_tasks, n_clouds, limit):
    """Clouds per task, their product at most `limit`."""
    out, prod = [], 1
    for _ in range(n_tasks):
        k = int(rng.integers(1, n_clouds + 1))
        while prod * k > limit:
            k -= 1
        out.append(k)
        prod *= k
    return out


@pytest.mark.parametrize('minimize_cost', [True, False])
def test_general_dags_reach_the_exact_optimum(minimize_cost):
    """Diamonds, fan-out / fan-in and random two-parent DAGs of 2-16 tasks,
    values >= 0: the device's objective, and the exact objective of the plan
    it returns, are within 1e-12 of the optimum (plans among equal optima
    are not compared). The TIME enumeration takes the largest finish time of
    any task, which is the reference's (leaves only) for values >= 0."""
    bad, n = [], 0
    for n_clouds in (1, 2, 3, 4, 6):
        store = _store(n_clouds)
        for shape in table_cases.DAG_SHAPES:
            for n_tasks in (2, 3, 4, 5, 7, 10, 13, 16):
                for regime in ('random', 'quantized', 'zeros', 'time'):
                    rng = np.random.default_rng(
                        [n_clouds, n_tasks, len(shape), len(regime),
                         int(minimize_cost)])
                    opts = _options(rng, n_tasks, n_clouds,
                                    4096 if minimize_cost else 2048)
                    tb = table_cases.dag(rng, regime, shape, n_tasks, n_clouds,
                                         options=opts)
                    chosen, obj, status = _device(store, tb, False,
                                                  minimize_cost)
                    best, _ = table_dp.dag_optimum(tb, minimize_cost)
                    n += 1
                    if status != 0:
                        bad.append((n_clouds, shape, n_tasks, regime, status))
                        continue
                    mine = table_dp.dag_objective(tb, chosen, minimize_cost)
                    for x in (obj, mine):
                        if not math.isclose(x, best, rel_tol=1e-12,
                                            abs_tol=1e-300):
                            bad.append((n_clouds, shape, n_tasks, regime,
                                        x, best))
    assert n == 5 * 3 * 8 * 4
    assert not bad, bad[:10]


def _frontier(tb):
    return table_dp.dag_optimum(tb, True, enumerate_limit=0)[0]


def test_enumeration_limits():
    """2^26 cloud assignments are enumerated on the device; one more task
    option, or a 17th task, returns status 2."""
    store4 = _store(4)
    rng = np.random.default_rng(26)
    tb = table_cases.dag(rng, 'random', 'random', 13, 4, options=[4] * 13)
    assert math.prod(len(r) for r in table_dp.representatives(tb)) == 2 ** 26
    chosen, obj, status = _device(store4, tb, False, True)
    assert status == 0
    best = _frontier(tb)
    assert math.isclose(obj, best, rel_tol=1e-12)
    assert math.isclose(table_dp.dag_objective(tb, chosen, True), best,
                        rel_tol=1e-12)
    # TIME at the limit: equal values, uniform tariffs -- every task in one
    # cloud is optimal (the longest path's values, no egress)
    tt = table_cases.dag(np.random.default_rng(27), 'time', 'diamond', 13, 4,
                         options=[4] * 13)
    chosen, obj, status = _device(store4, tt, False, False)
    one_cloud = [int(np.flatnonzero(c == 0)[0]) for c in tt.clouds]
    assert status == 0
    assert obj == table_dp.dag_objective(tt, one_cloud, False)
    assert table_dp.dag_objective(tt, chosen, False) == obj
    store6 = _store(6)
    above = table_cases.dag(np.random.default_rng(28), 'random', 'random', 13,
                            6, options=[4] * 12 + [5])
    assert _device(store6, above, False, True)[2] == 2
    assert _device(store6, above, False, False)[2] == 2
    big = table_cases.dag(np.random.default_rng(29), 'random', 'random', 17, 2,
                          options=[1] * 17)
    assert _device(_store(2), big, False, True)[2] == 2


def test_optimize_by_ilp_beyond_the_enumeration(monkeypatch):
    """_optimize_by_ilp on an 18-task DAG: the device returns status 2; COST
    takes dag_solver's answer, equal to the frontier optimum of the same
    tables; TIME raises OptimizerLimitError."""
    import skypilot_b200 as sky  # pylint: disable=import-outside-toplevel
    from skypilot_b200 import engine  # pylint: disable=import-outside-toplevel
    from skypilot_b200 import optimizer as opt_lib  # pylint: disable=import-outside-toplevel
    from tests import scenario_runner as runner  # pylint: disable=import-outside-toplevel
    from tests import scenarios  # pylint: disable=import-outside-toplevel
    runner.activate_catalog(scenarios.CATALOGS['bigdag'])
    sc = next(s for s in scenarios.big_dag_scenarios()
              if s['name'] == 'sparse18')
    calls = []
    real = engine.solve_tables

    def spy(store, *args, **kw):
        out = real(store, *args, **kw)
        calls.append((len(store.clouds), args, out))
        return out

    monkeypatch.setattr(engine, 'solve_tables', spy)
    O = opt_lib.Optimizer
    for minimize_cost in (True, False):
        dag, _ = runner.build_dag(sc)
        O._add_dummy_source_sink_nodes(dag)
        try:
            graph = dag.get_graph()
            topo = list(nx.topological_sort(graph))
            cost_map, _ = O._estimate_nodes_cost_or_time(topo, minimize_cost)
            if minimize_cost:
                _, objective = O._optimize_by_ilp(graph, topo, cost_map, True)
            else:
                with pytest.raises(sky.exceptions.OptimizerLimitError):
                    O._optimize_by_ilp(graph, topo, cost_map, False)
        finally:
            O._remove_dummy_source_sink_nodes(dag)
        n_clouds, args, (_, _, status) = calls[-1]
        assert status == 2
        if minimize_cost:
            tb = table_dp.Tables(*args[:5], n_clouds)
            assert math.isclose(objective, _frontier(tb), rel_tol=1e-12)


# ---- several DAGs in one launch ---------------------------------------------
def _solve_many(store, dags):
    """skyopt_solve_tables on several DAGs at once: [(Tables, is_chain,
    minimize_cost)] -> [(chosen, objective, status)]."""
    from skypilot_b200 import _native  # pylint: disable=import-outside-toplevel
    from skypilot_b200.engine import _addr  # pylint: disable=import-outside-toplevel
    n_clouds = len(store.clouds)
    values, clouds, tasks, par, tar, dag_rows = [], [], [], [], [], []
    for tb, is_chain, minimize_cost in dags:
        begin = len(tasks)
        for t in range(tb.n_tasks):
            row = {'n_parents': len(tb.parents[t]), 'parent_begin': len(par),
                   'edge_tariff_begin': len(tar), 'src_tariff_begin': -1}
            par.extend(tb.parents[t])
            for r in tb.edge_tariffs[t]:
                tar.extend(r.tolist())
            if tb.src_tariffs[t] is not None:
                row['src_tariff_begin'] = len(tar)
                tar.extend(tb.src_tariffs[t].tolist())
            tasks.append(row)
            values.append(tb.values[t])
            clouds.append(tb.clouds[t])
        dag_rows.append((begin, len(tasks), int(is_chain), int(minimize_cost)))
    n_tasks = len(tasks)
    offsets = np.zeros(n_tasks + 1, dtype=np.int64)
    offsets[1:] = np.cumsum([len(v) for v in values])
    flat_v = np.ascontiguousarray(np.concatenate(values), dtype=np.float64)
    flat_c = np.ascontiguousarray(np.concatenate(clouds), dtype=np.int32)
    task_a = np.zeros(n_tasks, dtype=_native.TASK_DTYPE)
    for i, row in enumerate(tasks):
        for k, v in row.items():
            task_a[k][i] = v
    dag_a = np.zeros(len(dags), dtype=_native.DAG_DTYPE)
    for i, (b, e, c, m) in enumerate(dag_rows):
        dag_a['task_begin'][i], dag_a['task_end'][i] = b, e
        dag_a['is_chain'][i], dag_a['minimize_cost'][i] = c, m
    par_a = np.asarray(par or [0], dtype=np.int32)
    tar_a = np.asarray(tar or [0.0], dtype=np.float64)
    assert len(tar) % n_clouds == 0
    chosen = np.zeros(n_tasks, dtype=np.int32)
    res = np.zeros(len(dags), dtype=_native.DAG_RESULT_DTYPE)
    lib = _native.load()
    _native.check(lib.skyopt_solve_tables(
        store.handle(0), _addr(flat_v), _addr(flat_c), _addr(offsets),
        _addr(task_a), n_tasks, _addr(par_a), len(par), _addr(tar_a),
        len(tar), _addr(dag_a), len(dags), _addr(chosen), _addr(res)))
    return [(chosen[b:e].tolist(), float(res['objective'][i]),
             int(res['status'][i])) for i, (b, e, _, _) in enumerate(dag_rows)]


def test_several_dags_in_one_launch():
    """Short chains on the lean recurrence, the general one (signed values)
    and the full evaluation (a hazard), a long chain, general DAGs (COST and
    TIME) and DAGs with an empty task, in one call: each equals its own
    single-DAG call and the model."""
    store = _store(4)
    rng = np.random.default_rng(41)
    c = table_cases.chain
    dags = [
        (c(rng, 'random', 8, 4), True, True),
        (c(rng, 'signed', 5, 4), True, True),
        (c(rng, 'hazard', 6, 4), True, True),
        (c(rng, 'quantized', 32, 4), True, False),
        (c(rng, 'random', 40, 4), True, True),
        (table_cases.dag(rng, 'random', 'diamond', 7, 4), False, True),
        (c(rng, 'random', 4, 4, empty_at=2), True, True),
        (table_cases.dag(rng, 'quantized', 'fan', 6, 4), False, False),
        (table_cases.dag(rng, 'random', 'random', 5, 4, empty_at=3), False,
         True),
        (c(rng, 'time', 1, 4), True, True),
    ]
    # general DAGs whose first, middle or last task has no candidate (the
    # first empty task is reported before the 16-task limit applies)
    dags += [(table_cases.dag(rng, 'random', 'random', n, 4, empty_at=at),
              False, True) for n, at in ((2, 0), (16, 8), (17, 16))]
    got = _solve_many(store, dags)
    for i, ((tb, is_chain, minimize_cost), g) in enumerate(zip(dags, got)):
        one = _device(store, tb, is_chain, minimize_cost)
        assert (g[0], g[1].hex(), g[2]) == (one[0], one[1].hex(), one[2]), i
        if tb.first_empty() is not None:
            assert g[2] == 1 and g[0] == [-1] * tb.n_tasks, i
        elif is_chain:
            plan, want = table_dp.chain_dp(tb)
            assert (g[0], g[1].hex(), g[2]) == (plan, want.hex(), 0), i
        else:
            best, _ = table_dp.dag_optimum(tb, minimize_cost)
            assert g[2] == 0 and math.isclose(g[1], best, rel_tol=1e-12), i
