"""Capacity reservations on the device against the reference's records
(tests/golden/reservations.json): every kernel mode and chain-DP path, a
session whose inventory changes, a batch mixing reservation and plain DAGs,
and a JobGroup."""
import pytest

import skypilot_b200 as sky
from skypilot_b200 import reservations
from skypilot_b200 import skypilot_config
from skypilot_b200.dag import DagExecution
from skypilot_b200.utils import registry
from tests import reservation_runner
from tests import reservation_scenarios
from tests import scenario_runner as runner
from tests import scenarios

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('mode', ['auto', 'fast-split', 'fast-noprune',
                                  'queue', 'tile'])
def test_records_match_reference_in_every_kernel_mode(mode):
    store = runner.activate_catalog(reservation_runner.golden()['catalog'])
    with runner.forced_paths(store, mode=mode):
        bad = reservation_runner.check_all()
    assert not bad, bad


@pytest.mark.parametrize('path', ['8', '32'])
def test_records_match_reference_on_every_chain_path(path):
    """The chain DP's full evaluation; the chain on the block that places
    the last task (runner.CHAIN_PATHS)."""
    with runner.forced_paths(chain=path):
        bad = reservation_runner.check_all()
    assert not bad, bad


def _plan(tasks):
    return [runner.res_record(t.best_resources) for t in tasks]


def _scenario(name):
    return next(s for s in reservation_scenarios.reservation_scenarios()
                if s['name'] == name)


def test_session_follows_inventory_changes():
    """Each call equals a fresh Optimizer.optimize under the inventory of
    that moment; a changed inventory re-solves from scratch."""
    runner.activate_catalog(reservation_scenarios.CATALOG)
    sc = _scenario('chain3_egress')
    inv = reservation_scenarios.RESERVATION_INVENTORY
    steps = [inv, [r for r in inv if r['name'] != 'cr-open-w2b'], [], inv]
    blocked = runner.blocked_list(
        {'blocked': [{'cloud': 'aws', 'zone': 'us-west-2b'}]})
    skypilot_config.set_config(sc['config'])
    try:
        dag, tasks = runner.build_dag(sc)
        with sky.Optimizer.session(dag) as session:
            for step in steps:
                reservations.set_reservations(step)
                for bl in (None, blocked):
                    session.optimize(bl)
                    got = _plan(tasks)
                    fresh_dag, fresh_tasks = runner.build_dag(sc)
                    sky.Optimizer.optimize(fresh_dag, blocked_resources=bl,
                                           quiet=True)
                    assert got == _plan(fresh_tasks), (step, bl)
    finally:
        reservations.set_reservations(None)
        skypilot_config.set_config(None)


def test_batch_mixing_reservation_and_plain_dags_equals_single_calls():
    runner.activate_catalog(reservation_scenarios.CATALOG)
    sc = _scenario('both_prio_v100_n5')
    skypilot_config.set_config(sc['config'])
    reservations.set_reservations(sc['reservations'])
    try:
        specs = [_scenario('aws_prio_v100_n4'), _scenario('chain3_egress'),
                 _scenario('aws_prio_spot_v100_n4'),
                 scenarios._single('azure_v100', cloud='azure',  # pylint: disable=protected-access
                                   accelerators='V100', num_nodes=3),
                 _scenario('gcp_prio_v100_n3')]
        built = [runner.build_dag(s) for s in specs]
        sky.Optimizer.optimize_batch([d for d, _ in built])
        batch = [_plan(tasks) for _, tasks in built]
        single = []
        for s in specs:
            dag, tasks = runner.build_dag(s)
            sky.Optimizer.optimize(dag, quiet=True)
            single.append(_plan(tasks))
        assert batch == single
        assert batch[0][0]['zone'] == 'us-west-2b'
    finally:
        reservations.set_reservations(None)
        skypilot_config.set_config(None)


def test_job_group_with_reservations():
    """The reference's SAME_INFRA score prices every node
    (sky/optimizer.py:1359-1360); AWS's launchables are per zone."""
    payload = reservation_runner.golden()
    rec = next(r for r in payload['records'] if r['name'] == 'jg_prio_two')
    case = _scenario('jg_prio_two')
    runner.activate_catalog(payload['catalog'])
    with reservation_runner.inventory_of(case):
        dag, tasks = runner.build_dag(case)
        dag.name = case['name']
        dag.set_execution(DagExecution.PARALLEL)
        sky.Optimizer.optimize_job_group(dag, quiet=True)
        plan = _plan(tasks)
        infras = {(p['cloud'], p['region']) for p in plan}
        assert len(infras) == 1
        assert list(infras.pop()) in rec['common_infras']
        # AWS launchables are per zone with reservations configured
        assert all(p['zone'] is not None for p in plan
                   if p['cloud'] in ('aws', 'gcp'))
        ours = sum(t.best_resources.get_cost(3600) * t.num_nodes
                   for t in tasks)
        dag_r, tasks_r = runner.build_dag(case)
        for t, p in zip(tasks_r, rec['plan']):
            # GCP prices the accelerator apart from the host VM
            accs = p['accelerators'] and {
                k: int(v) if float(v).is_integer() else v
                for k, v in p['accelerators'].items()}
            t.best_resources = sky.Resources(
                cloud=registry.CLOUD_REGISTRY.from_str(p['cloud']),
                instance_type=p['instance_type'], region=p['region'],
                zone=p['zone'], accelerators=accs, use_spot=p['use_spot'])
        del dag_r
        theirs = sum(t.best_resources.get_cost(3600) * t.num_nodes
                     for t in tasks_r)
        assert ours <= theirs + 1e-9
