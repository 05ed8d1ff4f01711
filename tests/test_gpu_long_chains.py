"""Chains longer than the fused chain DP's 32 tasks (step_kernel places them,
solve_kernel's per-candidate DP solves them), batches that mix them with
short chains and DAGs, and a catalog full of exact price ties: against the
reference's records, the oracle, and the exact table-level model
(oracle/table_dp.py) on the device's own candidate tables."""
import networkx as nx
import numpy as np
import pytest

import skypilot_b200 as sky
from oracle import optimizer_oracle as oo
from oracle import table_dp
from skypilot_b200 import engine
from skypilot_b200 import optimizer as opt_lib
from skypilot_b200 import workloads
from tests import scenario_runner as runner
from tests import scenarios

pytestmark = pytest.mark.gpu

_LONG = {sc['name']: sc for sc in scenarios.long_chain_scenarios()}


@pytest.mark.parametrize('name', sorted(_LONG))
def test_long_chain_matches_reference(name):
    """Ordered candidate tables, plan and objective of the unmodified
    reference (tests/golden/longchain.json)."""
    payload = runner.load_golden('longchain')
    assert payload['catalog'] == scenarios.CATALOGS['longchain']
    golden = next(r for r in payload['records'] if r['name'] == name)
    runner.activate_catalog(payload['catalog'])
    got = runner.run_scenario(_LONG[name])
    assert 'error' not in got, got
    diffs = runner.compare(golden, got, unordered_candidates=True)
    assert not diffs, diffs


def _problem(sc, store):
    minimize_cost = sc.get('minimize', 'cost') == 'cost'
    dag, _ = workloads.build_dag(sc)
    O = opt_lib.Optimizer
    O._add_dummy_source_sink_nodes(dag)  # pylint: disable=protected-access
    try:
        graph = dag.get_graph()
        topo = [t for t in nx.topological_sort(graph)
                if not opt_lib._is_dummy(t)]  # pylint: disable=protected-access
        b = engine.ProblemBuilder(store)
        O._state_problem(graph, topo, minimize_cost, [], True, builder=b)  # pylint: disable=protected-access
    finally:
        O._remove_dummy_source_sink_nodes(dag)  # pylint: disable=protected-access
    return b


def _model_tables(sol, n_tasks):
    """The device's own candidate tables, clouds and tariffs."""
    return table_dp.Tables(*opt_lib._dag_tables(sol, 0, n_tasks),  # pylint: disable=protected-access
                           len(sol.packed.store.clouds))


def _result(sol, n_tasks):
    """Plan as candidate records (a set's alternatives have no fixed order, so
    two builds of one DAG may list the same candidates in different order),
    objective bits and status."""
    return ([(int(c['inst_id']), int(c['region_id']), int(c['zone_id']))
             for c in sol.chosen[:n_tasks]],
            float(sol.dag[0]['objective']).hex(), int(sol.dag[0]['status']))


def _equals_model(sol, n_tasks):
    plan, objective = table_dp.chain_dp(_model_tables(sol, n_tasks))
    return (sol.chosen_index[:n_tasks].tolist(),
            float(sol.dag[0]['objective']).hex(),
            int(sol.dag[0]['status'])) == (plan, objective.hex(), 0)


@pytest.mark.parametrize('mode', ['auto', 'fast-split'])
def test_long_chains_equal_the_model_on_device_tables(mode):
    """33-, 40- (TIME) and 64-task chains (egress, inputs): one call, a
    session's re-solve and 50 launches of the device-resident loop give the
    model's plan and objective bits on the device's own tables."""
    store = runner.activate_catalog(scenarios.CATALOGS['longchain'])
    store.set_scan_mode(mode, 0)
    try:
        for name, sc in sorted(_LONG.items()):
            n = len(sc['tasks'])
            sol = engine.solve(_problem(sc, store), want_tables=True)
            assert _equals_model(sol, n), name
            got = _result(sol, n)
            sess = engine.Session(_problem(sc, store), device=0,
                                  want_tables=False)
            try:
                assert _result(sess.solution, n) == got, name
                assert _result(sess.resolve([]), n) == got, name
            finally:
                sess.close()
            timed, iter_ms, _ = engine.solve_timed(_problem(sc, store), 50,
                                                   False)
            assert len(iter_ms) == 50
            assert _result(timed, n) == got, name
    finally:
        store.set_scan_mode('auto', 0)


def test_mixed_batch_equals_one_dag_at_a_time():
    """optimize_batch of a 32-task chain, a 33-task chain, a diamond and
    single tasks: short chains then go through solve_kernel's minima fold,
    the long one through its per-candidate DP."""
    runner.activate_catalog(scenarios.CATALOGS['longchain'])
    basic = {s['name']: s for s in scenarios.basic_scenarios()}
    specs = [workloads.chain_scenario(32), _LONG['chain33'],
             basic['cfg3_diamond'],
             workloads.single('one_v100', accelerators='V100'),
             workloads.single('one_cpu', cpus='8+'),
             _LONG['chain64_egress_inputs']]
    built = [workloads.build_dag(sc) for sc in specs]
    sky.Optimizer.optimize_batch([d for d, _ in built])
    batch = [[workloads.res_record(t.best_resources) for t in ts]
             for _, ts in built]
    for sc, got in zip(specs, batch):
        dag, tasks = workloads.build_dag(sc)
        sky.Optimizer.optimize(dag, quiet=True)
        assert got == [workloads.res_record(t.best_resources)
                       for t in tasks], sc['name']


_TIED = dict(scenarios.CATALOGS['multi6k'], tie_suite=True)


def _tied_chains():
    return [sc for sc in scenarios.basic_scenarios()
            if oo._is_chain(len(sc['tasks']), sc.get('edges', []))  # pylint: disable=protected-access
            and not any(t.get('resources_kind') == 'list'
                        for t in sc['tasks'])]


@pytest.mark.parametrize('mode', ['auto', 'fast-split'])
def test_tied_catalog_chains_match_the_oracle(mode):
    """multi6k with prices on a two-decimal grid and no distinct-price
    guarantee: many exact ties within and across clouds. The oracle's stable
    sort applies the project's tie rule (the first CSV row); plan, ordered
    tables and objective must equal it, and the plan and objective bits the
    model on the device's tables (some of which tie across clouds)."""
    store = runner.activate_catalog(_TIED)
    store.set_scan_mode(mode, 0)
    n_ok = cross_ties = 0
    try:
        for sc in _tied_chains():
            want = oo.run_scenario(_TIED, sc)
            got = runner.run_scenario(sc)
            unordered = any(t.get('resources_kind') == 'set'
                            for t in sc['tasks'])
            diffs = runner.compare(want, got, unordered, check_message=False)
            assert not diffs, (sc['name'], diffs)
            if 'error' in want:
                continue
            n = len(sc['tasks'])
            sol = engine.solve(_problem(sc, store), want_tables=True)
            assert _equals_model(sol, n), sc['name']
            n_ok += 1
            tb = _model_tables(sol, n)
            for v, c in zip(tb.values, tb.clouds):
                mins = [v[c == g].min() for g in np.unique(c)]
                cross_ties += len(mins) != len(set(mins))
    finally:
        store.set_scan_mode('auto', 0)
    assert n_ok >= 10 and cross_ties

