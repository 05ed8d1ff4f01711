"""The fused step runs each chain DAG's DP on a block of its own, started from
the per-cloud minima as the task blocks publish them (skyopt_step.cuh), when
the grid holds one block per task and per DAG; else on the block that places
the DAG's last task. Both paths, several chain blocks in one launch, and the
hand-off counters across the launches of the device-resident loop."""
import networkx as nx
import numpy as np
import pytest

import skypilot_b200 as sky
from skypilot_b200 import _native
from skypilot_b200 import engine
from skypilot_b200 import optimizer as opt_lib
from skypilot_b200 import workloads
from tests import scenario_runner as runner
from tests import scenarios

pytestmark = pytest.mark.gpu

_POOL = [
    {'accelerators': 'V100'}, {'accelerators': 'T4'}, {'accelerators': 'L4'},
    {'accelerators': 'A100:8'}, {'accelerators': 'H100:8'}, {'cpus': '8+'},
    {'cpus': '32+', 'memory': '128+'}, {'accelerators': 'A10G'},
    {'accelerators': 'T4:4', 'use_spot': True}, {'cpus': '4+', 'use_spot': True},
    {'accelerators': 'K80'}, {'memory': '64+'},
]


@pytest.mark.parametrize('path', ['32', '40'])
def test_chain_on_last_task_block_agrees_with_reference(path):
    """32 keeps every chain DP on the block that places the DAG's last task
    (the path of batches with more tasks and DAGs than the grid holds), 40
    adds the full evaluation: the multi6k and fuzz6k chain suites still give
    the reference's records."""
    bad, forms = runner.check_chain_suites(chain=path)
    assert not bad, bad
    assert forms


def _random_chain(rng, name):
    specs = []
    for _ in range(int(rng.integers(2, 7))):
        spec = dict(_POOL[int(rng.integers(len(_POOL)))])
        if rng.uniform() < 0.8:
            spec['outputs_gb'] = float(rng.choice([0.5, 20, 300, 2500]))
        if rng.uniform() < 0.3:
            spec['num_nodes'] = 2
        specs.append(spec)
    return workloads.chain(name, specs)


def _state(dag, builder):
    opt_lib.Optimizer._add_dummy_source_sink_nodes(dag)  # pylint: disable=protected-access
    try:
        graph = dag.get_graph()
        topo = [t for t in nx.topological_sort(graph)
                if not opt_lib._is_dummy(t)]  # pylint: disable=protected-access
        return opt_lib.Optimizer._state_problem(  # pylint: disable=protected-access
            graph, topo, True, [], True, builder=builder)
    finally:
        opt_lib.Optimizer._remove_dummy_source_sink_nodes(dag)  # pylint: disable=protected-access


def _plan(sol, first_task, n_tasks, dag_index):
    d = sol.dag[dag_index]
    out = {'status': int(d['status']), 'task_fail': int(d['task_fail'])}
    if out['status'] == 0:
        c = sol.chosen[first_task:first_task + n_tasks]
        out['objective'] = float(d['objective']).hex()
        out['index'] = sol.chosen_index[first_task:first_task + n_tasks].tolist()
        out['cands'] = [(int(x['inst_id']), int(x['region_id']),
                         int(x['zone_id']), float(x['hourly']).hex(),
                         float(x['value']).hex()) for x in c]
    return out


def test_several_chain_blocks_match_one_dag_at_a_time():
    """Sixteen chain DAGs (2-6 tasks, egress between them, one with a task
    nothing satisfies) in one fused launch, each chain DP on its own block,
    equal the same DAGs solved one per call: plans, candidate records and
    objectives bit for bit. So do they with every chain DP forced onto the
    block that places its DAG's last task, a launch without the chain
    blocks: the eight chains of one instance type keep the scan's pieces
    fewer than the tasks and DAGs, so that launch is smaller."""
    store = runner.activate_catalog(scenarios.CATALOGS['multi6k'])
    rng = np.random.default_rng(11)
    chains = [_random_chain(rng, f'c{i}') for i in range(7)]
    chains.insert(3, workloads.chain('c_empty', [{'accelerators': 'V100'},
                                                 {'cpus': '100000+'},
                                                 {'accelerators': 'T4'}]))
    pinned = {'cloud': 'aws', 'instance_type': 'p3.2xlarge', 'outputs_gb': 20}
    chains += [workloads.chain(f'p{i}', [pinned] * 4) for i in range(8)]
    for path in (None, '32'):
        with runner.forced_paths(chain=path):
            # an unknown flag is refused and leaves the setting as it was
            assert _native.load().skyopt_set_chain_paths(8) == -1
            batch = engine.ProblemBuilder(store)
            sizes = []
            for sc in chains:
                dag, tasks = workloads.build_dag(sc)
                _state(dag, batch)
                sizes.append(len(tasks))
            sol = engine.solve(batch)
            stats = engine.LAST_STATS
            assert int(stats.scan_form) == 4
            assert int(stats.total_launches) == 1
            if path is None:
                # a block per task and one per DAG
                assert int(stats.scan_blocks) >= sum(sizes) + len(sizes)
            else:
                assert int(stats.scan_blocks) < sum(sizes) + len(sizes)
            first = 0
            statuses = []
            for i, (sc, n) in enumerate(zip(chains, sizes)):
                one = engine.ProblemBuilder(store)
                dag, _ = workloads.build_dag(sc)
                _state(dag, one)
                want = _plan(engine.solve(one), 0, n, 0)
                assert _plan(sol, first, n, i) == want, (path, sc['name'])
                statuses.append(want['status'])
                first += n
        assert statuses.count(0) >= 14 and statuses[3] == 1


def test_device_resident_loop_rearms_the_hand_off():
    """Three hundred launches of the device-resident loop on one chain (the
    hand-off words are zeroed by the chain blocks, never by the host between
    launches) give the plan and objective of a single call."""
    store = runner.activate_catalog(scenarios.CATALOGS['multi6k'])
    sc = workloads.chain('loop', [{'accelerators': 'V100', 'outputs_gb': 300},
                                  {'cpus': '8+', 'outputs_gb': 20},
                                  {'accelerators': 'A100:8', 'outputs_gb': 2500},
                                  {'accelerators': 'T4'}])
    one = engine.ProblemBuilder(store)
    dag, _ = workloads.build_dag(sc)
    _state(dag, one)
    want = _plan(engine.solve(one), 0, 4, 0)
    assert want['status'] == 0
    loop = engine.ProblemBuilder(store)
    dag, _ = workloads.build_dag(sc)
    _state(dag, loop)
    sol, iter_ms, _ = engine.solve_timed(loop, 300, False)
    assert len(iter_ms) == 300 and np.all(iter_ms > 0)
    assert int(sol.stats.scan_form) == 4
    assert _plan(sol, 0, 4, 0) == want
