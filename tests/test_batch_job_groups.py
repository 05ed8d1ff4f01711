"""JobGroups on the batch path without a GPU: how a group is stated as one
SAME_INFRA DAG, that `job_groups=False` leaves a batch's statement as it
was, which groups are left to the host, and the C ABI of the new kind."""
import ctypes
import os
import re

import pytest

from skypilot_b200 import _native
from skypilot_b200 import engine
from skypilot_b200 import optimizer as opt_lib
from skypilot_b200.dag import DagExecution
from tests import scenario_runner as runner
from tests import scenarios

_REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def store():
    return runner.activate_catalog(scenarios.CATALOGS['multi6k'])


def _group(specs, name='jg', edges=(), parallel=True):
    tasks = []
    for i, spec in enumerate(specs):
        spec = dict(spec)
        extra = {k: spec.pop(k) for k in ('num_nodes', 'time_est', 'inputs')
                 if k in spec}
        kind = spec.pop('kind', 'single')
        resources = spec.pop('alts', [spec])
        tasks.append(dict(name=f'{name}_job{i}', resources=resources,
                          resources_kind=kind, **extra))
    dag, made = runner.build_dag(dict(name=name, tasks=tasks,
                                      edges=list(edges)))
    dag.name = name
    if parallel:
        dag.set_execution(DagExecution.PARALLEL)
    return dag, made


_SPECS = [
    dict(accelerators='V100', inputs=['s3://bucket/data', 40.0]),
    dict(cpus='8+', num_nodes=3),
    dict(accelerators='T4', cloud='gcp', inputs=['gs://bucket/d', 5.0]),
    dict(cpus='4+', use_spot=True),
]


def test_group_is_one_same_infra_dag(store):
    """Kind 2, the jobs in `dag.tasks` order, no parents even where the
    group has edges, and a source tariff row for every job with inputs."""
    del store
    dag, tasks = _group(_SPECS, edges=[(0, 1), (1, 3)])
    batch = opt_lib._Batch([dag], True, [0], [[]], job_groups=True)  # pylint: disable=protected-access
    b = batch.builders[0]
    assert len(b.dags) == 1
    d = b.dags[0]
    assert d['is_chain'] == _native.DAG_SAME_INFRA == 2
    assert (d['task_begin'], d['task_end']) == (0, len(tasks))
    assert batch.problems[0].tasks == tasks
    for j, t in enumerate(b.tasks):
        assert t['n_parents'] == 0
        assert (t['src_tariff_begin'] >= 0) == ('inputs' in _SPECS[j])
    packed = b.pack()
    assert int(packed.dags['is_chain'][0]) == 2
    assert list(packed.tasks['n_parents'][:len(tasks)]) == [0] * len(tasks)


@pytest.mark.parametrize('minimize_cost', [True, False])
def test_each_job_is_stated_as_its_single_task_dag(store, minimize_cost):
    """The queries, slots, costs, task records and tariffs of the group are
    those of the jobs stated one by one as single-task DAGs into one
    builder, as optimize_job_group stated them before; only the DAG records
    and the blocked copies (one per job there) differ."""
    blocked = [runner.blocked_list(dict(blocked=[dict(cloud='aws',
                                                      region='us-east-1')]))]
    dag, tasks = _group(_SPECS)
    batch = opt_lib._Batch([dag], minimize_cost, [0], blocked,  # pylint: disable=protected-access
                           job_groups=True)
    b = batch.builders[0]
    ref = engine.ProblemBuilder(store)
    for task in tasks:
        graph = opt_lib.nx.DiGraph()
        graph.add_node(task)
        opt_lib.Optimizer._state_problem(graph, [task], minimize_cost,  # pylint: disable=protected-access
                                         blocked[0], True, builder=ref)
    assert b.query_recs == ref.query_recs
    assert b.slot_recs == ref.slot_recs
    assert b.slot_cost == ref.slot_cost
    assert b.task_recs == ref.task_recs
    assert b.tariffs == ref.tariffs
    assert b.blocked == ref.blocked[:len(b.blocked)]
    assert len(ref.blocked) == len(tasks) * len(b.blocked)


@pytest.mark.parametrize('n_devices', [1, 2])
def test_job_groups_off_packs_as_before(store, n_devices):
    """Without `job_groups` a JobGroup is stated like any DAG: the packed
    problem equals that of the same DAGs without PARALLEL execution."""
    del store

    def dags(parallel):
        out = []
        for k in range(5):
            specs = (_SPECS[k % 4:] + _SPECS[:k % 4])[:2 + k % 3]
            edges = [(0, 1)] if len(specs) == 2 else [(0, 1), (0, 2)]
            out.append(_group(specs, name=f'g{k}', edges=edges,
                              parallel=parallel and k != 2)[0])
        return out

    def packed(batch):
        out = []
        for b in batch.builders:
            p = b.pack()
            out.append([bytes(getattr(p, f)) for f in (
                'queries', 'slots', 'tasks', 'dags', 'blocked', 'parents',
                'tariffs')])
        return out

    lists = [[] for _ in range(5)]
    devices = list(range(n_devices))
    off = opt_lib._Batch(dags(True), True, devices, lists)  # pylint: disable=protected-access
    plain = opt_lib._Batch(dags(False), True, devices, lists)  # pylint: disable=protected-access
    assert packed(off) == packed(plain)
    assert not off.groups
    on = opt_lib._Batch(dags(True), True, devices, lists, job_groups=True)  # pylint: disable=protected-access
    assert on.groups == {0, 1, 3, 4}
    kinds = [int(d['is_chain']) for b in on.builders for d in b.dags]
    assert kinds.count(_native.DAG_SAME_INFRA) == 4


def test_estimator_and_ordered_groups_go_to_the_host(store):
    """A group with a time estimator is scored by a Python callback: it is
    left out of the device problem, and a session handles it on the host.
    A session also redoes a group with ordered resources on the host (its
    choice depends on the blocked list), as it does for any such DAG."""
    del store
    est, _ = _group([dict(accelerators='V100'),
                     dict(cpus='8+', time_est={'default': 7200})], name='est')
    ordered, _ = _group([dict(kind='list', alts=[dict(accelerators='A100:8'),
                                                 dict(accelerators='V100')]),
                         dict(cpus='8+')], name='ordered')
    plain, _ = _group([dict(accelerators='T4')], name='plain')
    dags = [est, ordered, plain]
    batch = opt_lib._Batch([est, plain], True, [0], [[], []],  # pylint: disable=protected-access
                           job_groups=True)
    assert batch.host_groups == {0}
    assert batch.shards == [[1]]
    assert [d['is_chain'] for d in batch.builders[0].dags] == [2]
    session = opt_lib.BatchOptimizerSession(dags, job_groups=True)
    assert session._fallback == {0, 1}  # pylint: disable=protected-access
    assert opt_lib.BatchOptimizerSession(dags)._fallback == {1}  # pylint: disable=protected-access


def test_dag_kind_in_header_exports_and_signature():
    with open(os.path.join(_REPO, 'include', 'skyopt.h'),
              encoding='utf-8') as f:
        header = f.read()
    assert re.search(r'#define SKYOPT_DAG_SAME_INFRA 2\b', header)
    assert re.search(r'int skyopt_dag_kinds\(void\);', header)
    assert 'skyopt_dag_kinds' in _native.EXPORTS
    assert _native.ABI_VERSION == 4
    lib = _native.load()
    assert lib.skyopt_dag_kinds.restype is ctypes.c_int
    assert lib.skyopt_dag_kinds() == _native.DAG_SAME_INFRA
