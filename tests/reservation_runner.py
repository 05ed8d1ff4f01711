"""Runs the reservation scenarios (tests/reservation_scenarios.py)
through skypilot_b200 and compares them with the reference's records
(tests/golden/reservations.json) exactly: plan, ordered candidate tables with
bit-equal values, and the DP objective, which with reservations is not the
plan's total cost (_compute_total_cost prices every node)."""
import contextlib
from typing import Any, Dict, List

import networkx as nx

from skypilot_b200 import optimizer as opt_lib
from skypilot_b200 import reservations
from skypilot_b200 import skypilot_config
from tests import reservation_scenarios
from tests import scenario_runner as runner


def golden() -> Dict[str, Any]:
    payload = runner.load_golden('reservations')
    assert payload['catalog'] == reservation_scenarios.CATALOG
    return payload


def optimizer_scenarios() -> List[Dict[str, Any]]:
    return [s for s in reservation_scenarios.reservation_scenarios()
            if s.get('kind') != 'job_group']


@contextlib.contextmanager
def inventory_of(scenario):
    """The scenario's SkyPilot config and reservation inventory."""
    skypilot_config.set_config(scenario.get('config'))
    reservations.set_reservations(scenario.get('reservations'))
    try:
        yield
    finally:
        reservations.set_reservations(None)
        skypilot_config.set_config(None)


def run(scenario) -> Dict[str, Any]:
    """Candidates and plan as scenario_runner records them, plus the
    objective of the reference's DP over those candidates."""
    inner = {k: v for k, v in scenario.items() if k != 'config'}
    with inventory_of(scenario):
        record = runner.run_scenario(inner)
        if 'error' in record:
            return record
        dag, tasks = runner.build_dag(scenario)
        minimize_cost = scenario.get('minimize', 'cost') == 'cost'
        Optimizer = opt_lib.Optimizer
        Optimizer._add_dummy_source_sink_nodes(dag)  # pylint: disable=protected-access
        try:
            graph = dag.get_graph()
            topo = list(nx.topological_sort(graph))
            cost_map, _ = Optimizer._estimate_nodes_cost_or_time(  # pylint: disable=protected-access
                topo, minimize_cost, runner.blocked_list(scenario), quiet=True)
            if dag.is_chain():
                plan, objective = Optimizer._optimize_by_dp(  # pylint: disable=protected-access
                    topo, cost_map, minimize_cost)
            else:
                plan, objective = Optimizer._optimize_by_ilp(  # pylint: disable=protected-access
                    graph, topo, cost_map, minimize_cost)
        finally:
            Optimizer._remove_dummy_source_sink_nodes(dag)  # pylint: disable=protected-access
        record['objective'] = float(objective)
        record['dp_plan'] = [runner.res_record(plan[t]) for t in tasks]
    return record


def diffs(gold: Dict[str, Any], got: Dict[str, Any]) -> List[str]:
    out: List[str] = []
    if 'error' in gold or 'error' in got:
        if gold.get('error') != got.get('error'):
            out.append(f'error: {gold.get("error")} vs {got.get("error")}')
        return out
    if got['candidates'] != gold['candidates']:
        for ti, (g, o) in enumerate(zip(gold['candidates'],
                                        got['candidates'])):
            if g != o:
                first = next((i for i, (a, b) in enumerate(zip(g, o))
                              if a != b), min(len(g), len(o)))
                out.append(f'task {ti}: {len(g)} vs {len(o)} candidates, '
                           f'first difference at {first}')
    for key in ('plan', 'dp_plan'):
        if got[key] != gold['plan']:
            out.append(f'{key}: {gold["plan"]} vs {got[key]}')
    # chains: the reference's DP operation by operation; general DAGs: the
    # exact optimum, summed in another order
    if (got['objective'] != gold['objective'] if gold['is_chain'] else
            not runner.close(gold['objective'], got['objective'])):
        out.append(f'objective: {gold["objective"]!r} vs {got["objective"]!r}')
    for key in ('total_cost', 'total_time'):
        if not runner.close(gold[key], got[key]):
            out.append(f'{key}: {gold[key]} vs {got[key]}')
    return out


def check_all() -> List[Any]:
    """Every optimizer record of the fixture; the differences found."""
    payload = golden()
    records = {r['name']: r for r in payload['records']}
    runner.activate_catalog(payload['catalog'])
    bad = []
    for sc in optimizer_scenarios():
        d = diffs(records[sc['name']], run(sc))
        if d:
            bad.append((sc['name'], d[:3]))
    return bad
