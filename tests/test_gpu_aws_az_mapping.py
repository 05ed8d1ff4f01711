"""The AWS account's zone mapping on the device, against the reference's
records on the mapped `azmap` catalog (tests/golden/azmap.json,
tests/golden/azmap_reservations.json): every kernel mode and chain-DP path,
a session whose blocked zone names grow, a batch across the mapped store,
the accelerator listing and a JobGroup."""
import pytest

import skypilot_b200 as sky
from skypilot_b200 import reservations
from skypilot_b200 import skypilot_config
from skypilot_b200.dag import DagExecution
from tests import azmap_runner
from tests import azmap_scenarios
from tests import scenario_runner as runner
from tests.test_oracle_listing import normalise

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('mode', ['auto', 'fast-split', 'fast-noprune',
                                  'queue', 'tile'])
def test_records_match_reference_in_every_kernel_mode(mode):
    with runner.forced_paths(azmap_runner.activate(), mode=mode):
        bad = azmap_runner.check_all()
    assert not bad, bad


@pytest.mark.parametrize('path', ['8', '32'])
def test_records_match_reference_on_every_chain_path(path):
    """The chain DP's full evaluation; the chain on the block that places
    the last task (runner.CHAIN_PATHS)."""
    with runner.forced_paths(chain=path):
        bad = azmap_runner.check_all()
    assert not bad, bad


def _plan(tasks):
    return [runner.res_record(t.best_resources) for t in tasks]


def _scenario(name):
    return next(s for s in azmap_runner.optimizer_scenarios()
                if s['name'] == name)


def test_session_with_growing_blocked_zone_names():
    """Each call equals a fresh Optimizer.optimize with the same blocked
    list; the failover walks the account's zone names."""
    azmap_runner.activate()
    sc = _scenario('spot_aws_t4')
    dag, tasks = runner.build_dag(sc)
    blocked = []
    seen = []
    with sky.Optimizer.session(dag) as session:
        for _ in range(6):
            bl = runner.blocked_list({'blocked': blocked}) if blocked else None
            session.optimize(bl)
            got = _plan(tasks)
            fresh_dag, fresh_tasks = runner.build_dag(sc)
            sky.Optimizer.optimize(fresh_dag, blocked_resources=bl,
                                   quiet=True)
            assert got == _plan(fresh_tasks), blocked
            aws = [p for p in got if p['cloud'] == 'aws']
            if not aws:
                break
            zone = aws[0]['zone']
            assert zone is not None and not zone.startswith(
                tuple(azmap_scenarios.UNMAPPED_REGIONS))
            assert '-az' not in zone
            seen.append(zone)
            # what the failover loop blocks: the failed spot zone
            blocked.append({'cloud': 'aws', 'zone': zone, 'use_spot': True})
    assert len(set(seen)) == len(seen) >= 2


def test_batch_across_the_mapped_store_equals_single_calls():
    azmap_runner.activate()
    names = ['v100', 'spot_aws_t4', 'zone_name', 'chain3_egress',
             'diamond_egress', 'resv_v100_n4']
    specs = [_scenario(n) for n in names]
    resv = _scenario('resv_v100_n4')
    blocked = runner.blocked_list(_scenario('blocked_zones'))
    skypilot_config.set_config(resv['config'])
    reservations.set_reservations(resv['reservations'])
    try:
        for bl in (None, blocked):
            built = [runner.build_dag(s) for s in specs]
            sky.Optimizer.optimize_batch([d for d, _ in built],
                                         blocked_resources=bl)
            batch = [_plan(tasks) for _, tasks in built]
            single = []
            for s in specs:
                dag, tasks = runner.build_dag(s)
                sky.Optimizer.optimize(dag, blocked_resources=bl, quiet=True)
                single.append(_plan(tasks))
            assert batch == single
            zones = [p['zone'] for plan in batch for p in plan
                     if p['cloud'] == 'aws' and p['zone'] is not None]
            assert zones and not any('-az' in z for z in zones)
    finally:
        reservations.set_reservations(None)
        skypilot_config.set_config(None)


@pytest.mark.parametrize('case', azmap_scenarios.listing_cases(),
                         ids=lambda c: c['name'])
def test_listing_matches_reference(case):
    rec = azmap_runner.records()[case['name']]
    azmap_runner.activate()
    got = sky.catalog.list_accelerators(**case['kwargs'])
    as_lists = {k: [list(i) for i in v] for k, v in got.items()}
    assert list(got.keys()) == rec['order']
    assert normalise(as_lists) == rec['listing']


@pytest.mark.parametrize('case', azmap_scenarios.job_group_cases(),
                         ids=lambda c: c['name'])
def test_job_group(case):
    rec = azmap_runner.records()[case['name']]
    azmap_runner.activate()
    dag, tasks = runner.build_dag(case)
    dag.name = case['name']
    dag.set_execution(DagExecution.PARALLEL)
    sky.Optimizer.optimize_job_group(dag, quiet=True)
    plan = _plan(tasks)
    infras = {(p['cloud'], p['region']) for p in plan}
    assert len(infras) == 1
    assert list(infras.pop()) in rec['common_infras']
    if len(rec['common_infras']) == 1:
        assert plan == rec['plan']
