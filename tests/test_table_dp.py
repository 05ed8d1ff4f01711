"""CPU tests of the exact table-level model (oracle/table_dp.py) that the GPU
tests of skyopt_solve_tables compare against: it reproduces the oracle's
chain DP (itself pinned by the reference's records, test_oracle.py) on every
golden chain scenario, its vectorised form equals the literal per-candidate
loop, and each regime of tests/table_cases.py tells a correct DP from one
with a subtle bug ("mutants") -- so the GPU tests would catch a kernel that
made that mistake."""
import math
import operator

import numpy as np
import pytest

from oracle import optimizer_oracle as oo
from oracle import table_dp
from tests import table_cases
from tests import scenarios
from tests import scenario_runner as runner
from tests.test_oracle import _cases


def _tables_of(tasks, tables, minimize_cost):
    """The oracle's candidate tables ([(launchable, value)] per task) in the
    layout of engine.solve_tables."""
    names = sorted({c['cloud'] for rows in tables for c, _ in rows})
    values = [[v for _, v in rows] for rows in tables]
    clouds = [[names.index(c['cloud']) for c, _ in rows] for rows in tables]
    edges, srcs = [], []
    for i, task in enumerate(tasks):
        if i == 0:
            edges.append([])
            srcs.append(None if task.get('inputs') is None else [
                oo.edge_value(minimize_cost, None, None, task, {'cloud': n})
                for n in names])
        else:
            nbytes = tasks[i - 1].get('outputs_gb')
            # egress out of the parent's cloud into any other one
            edges.append([[oo.egress(minimize_cost, n, '-', nbytes)
                           for n in names]])
            srcs.append(None)
    parents = [[i - 1] if i else [] for i in range(len(tasks))]
    return table_dp.Tables(values, clouds, parents, edges, srcs, len(names))


def _chain_cases():
    out = [p for p in _cases()
           if oo._is_chain(len(p.values[1]['tasks']),  # pylint: disable=protected-access
                           p.values[1].get('edges', []))]
    for sc in scenarios.long_chain_scenarios():
        out.append(pytest.param('longchain', sc, id=f'longchain:{sc["name"]}'))
    return out


@pytest.mark.parametrize('catalog,scenario', _chain_cases())
def test_model_matches_oracle_chain_dp(catalog, scenario, monkeypatch):
    """Same plan indices and the same objective bits as
    optimizer_oracle.optimize_by_dp on the oracle's own tables."""
    seen = []
    real = oo.optimize_by_dp

    def check(tasks, tables, minimize_cost):
        plan, objective = real(tasks, tables, minimize_cost)
        tb = _tables_of(tasks, tables, minimize_cost)
        for fn in (table_dp.chain_dp, table_dp.chain_dp_loop):
            got_plan, got_obj = fn(tb)
            assert got_plan == plan, fn.__name__
            assert float(got_obj).hex() == float(objective).hex(), fn.__name__
        seen.append(len(tasks))
        return plan, objective

    monkeypatch.setattr(oo, 'optimize_by_dp', check)
    spec = (runner.load_golden(catalog)['catalog'] if catalog != 'longchain'
            else scenarios.CATALOGS['longchain'])
    record = oo.run_scenario(spec, scenario)
    assert seen or 'error' in record


def _same(a, b):
    return a[0] == b[0] and float(a[1]).hex() == float(b[1]).hex()


def _small(seed, regime):
    rng = np.random.default_rng([seed, table_cases.CHAIN_REGIMES.index(regime)])
    return table_cases.chain(rng, regime, int(rng.integers(1, 7)),
                             int(rng.integers(1, 5)))


@pytest.mark.parametrize('regime', table_cases.CHAIN_REGIMES)
def test_vectorised_model_equals_the_loop(regime):
    for seed in range(60):
        tb = _small(seed, regime)
        assert _same(table_dp.chain_dp(tb), table_dp.chain_dp_loop(tb)), seed


def test_signed_zero_chains():
    """The reference's answers on the crafted +-0.0 chains: the first of two
    equal parent sums, and a +0.0 objective."""
    for n_clouds in (2, 5):
        first, *alternating = table_cases.signed_zero_chains(n_clouds)
        for tb in [first] + alternating:
            assert _same(table_dp.chain_dp(tb), table_dp.chain_dp_loop(tb))
        plan, obj = table_dp.chain_dp(first)
        assert (plan, obj.hex()) == ([0, 0], '0x0.0p+0')
        for tb in alternating:
            _, obj = table_dp.chain_dp(tb)
            assert obj.hex() == '0x0.0p+0'


# ---- mutants: chain DPs with one subtle bug each ---------------------------
def _per_cloud(tb, lean: bool):
    """The C-wide recurrence over per-(task, cloud) representatives. lean:
    the representative is the first candidate of the smallest VALUE and no
    hazard test follows (a pricier candidate in front whose sum rounds the
    same is missed). Else the exact first minimum of dp within the cloud,
    but ties across clouds go to the smaller cloud number."""
    dp, back = None, []
    for t in range(tb.n_tasks):
        v, cl = tb.values[t], tb.clouds[t]
        if t == 0:
            src = tb.src_tariffs[0]
            best = {int(h): (0.0 + (float(src[h]) if src is not None else 0.0), 0)
                    for h in np.unique(cl)}
        else:
            pcl = tb.clouds[t - 1]
            tar = tb.edge_tariffs[t][0]
            reps = {}
            for p in range(len(pcl)):
                g = int(pcl[p])
                key = tb.values[t - 1][p] if lean else dp[p]
                if g not in reps or key < reps[g][0]:
                    reps[g] = (key, p)
            best = {}
            for h in np.unique(cl):
                cands = []
                for g, (_, p) in reps.items():
                    s = dp[p] + (0.0 if g == h else float(tar[g]))
                    cands.append((s, p if lean else g, p))
                s, _, p = min(cands)
                best[int(h)] = (s, p)
        dp = np.array([v[i] + best[int(cl[i])][0] for i in range(len(v))])
        back.append([best[int(cl[i])][1] for i in range(len(v))])
    reps = {}
    for i in range(len(dp)):
        g = int(tb.clouds[-1][i])
        key = tb.values[-1][i] if lean else dp[i]
        if g not in reps or key < reps[g][0]:
            reps[g] = (key, i)
    obj, _, idx = min((dp[i] + 0.0, i if lean else g, i)
                      for g, (_, i) in reps.items())
    plan = [0] * tb.n_tasks
    for t in range(tb.n_tasks - 1, -1, -1):
        plan[t] = idx
        idx = back[t][idx]
    return plan, 0.0 + obj


loop = table_dp.chain_dp_loop
MUTANTS = {
    # name: (mutant, the regime that must expose it)
    'no_hazard_fallback': (lambda tb: _per_cloud(tb, True), 'hazard'),
    'le_instead_of_lt': (lambda tb: loop(tb, take=operator.le), 'quantized'),
    'cross_cloud_ties_by_cloud': (lambda tb: _per_cloud(tb, False), 'time'),
    'same_cloud_egress': (lambda tb: loop(tb, same_cloud_egress=True),
                          'random'),
    'last_minimum_sink': (lambda tb: loop(tb, sink_take=operator.le),
                          'quantized'),
}


@pytest.mark.parametrize('name', sorted(MUTANTS))
def test_regime_exposes_mutant(name):
    mutant, regime = MUTANTS[name]
    caught = 0
    for seed in range(40):
        tb = _small(seed, regime)
        if not _same(mutant(tb), table_dp.chain_dp(tb)):
            caught += 1
    assert caught, f'{name}: no {regime} case tells it from the model'


# ---- general DAGs ----------------------------------------------------------
@pytest.mark.parametrize('minimize_cost', [True, False])
def test_dag_optimum_matches_the_oracle_enumeration(minimize_cost):
    """dag_optimum on a chain equals the chain DP's objective (COST within
    rounding; TIME exactly), and the frontier DP equals the enumeration."""
    for seed in range(30):
        rng = np.random.default_rng(seed)
        tb = table_cases.chain(rng, 'random', int(rng.integers(1, 5)),
                               int(rng.integers(1, 4)))
        best, plan = table_dp.dag_optimum(tb, minimize_cost)
        assert table_dp.dag_objective(tb, plan, minimize_cost) == best
        if minimize_cost:
            _, obj = table_dp.chain_dp(tb)
            assert math.isclose(best, obj, rel_tol=1e-12)
            big, _ = table_dp.dag_optimum(tb, True, enumerate_limit=0)
            assert math.isclose(best, big, rel_tol=1e-12)
