"""Capacity reservations without a GPU: the oracle against the reference's
records (tests/golden/reservations.json), the consumption rules and their
configuration, AWS's per-zone split and the device table's layout."""
import numpy as np
import pytest

from oracle import reservation_oracle
from skypilot_b200 import _native
from skypilot_b200 import reservations
from skypilot_b200 import skypilot_config
from skypilot_b200.clouds import aws as aws_lib
from skypilot_b200.clouds import gcp as gcp_lib
from tests import reservation_runner
from tests import reservation_scenarios
from tests import scenario_runner as runner

R = reservations.Reservation


@pytest.fixture(autouse=True)
def _clean():
    yield
    reservations.set_reservations(None)
    reservations.set_provider(None)
    skypilot_config.set_config(None)


@pytest.mark.parametrize('scenario', reservation_runner.optimizer_scenarios(),
                         ids=lambda s: s['name'])
def test_oracle_reproduces_reference_record(scenario):
    payload = reservation_runner.golden()
    gold = next(r for r in payload['records'] if r['name'] == scenario['name'])
    got = reservation_oracle.run_scenario(payload['catalog'], scenario)
    assert got.get('error') == gold.get('error')
    if 'error' in gold:
        return
    assert got['candidates'] == gold['candidates']
    assert got['plan'] == gold['plan']
    assert runner.close(got['objective'], gold['objective'])
    if gold['is_chain']:
        assert got['objective'] == gold['objective']
    assert runner.close(got['total_cost'], gold['total_cost'])
    assert runner.close(got['total_time'], gold['total_time'])


def test_fixture_has_plans_that_reservations_flip():
    records = {r['name']: r for r in reservation_runner.golden()['records']}
    assert records['aws_prio_v100_n4']['objective'] == 0.0
    assert records['aws_prio_v100_n4']['plan'][0]['zone'] == 'us-west-2b'
    # partial coverage: 6 nodes, 4 reserved
    assert records['aws_prio_v100_n6_partial']['objective'] == 2 * 3.264
    assert records['gcp_specific_v100_n8']['plan'][0]['zone'] == 'us-west1-b'


def _inventory():
    return [R('aws', 'p3.2xlarge', 'us-west-2b', 'open', 4),
            R('aws', 'p3.2xlarge', 'us-west-2b', 'tgt', 8, targeted=True),
            R('aws', 'p3.2xlarge', 'us-west-2b', 'open', 2),  # same name
            R('gcp', 'n1-highmem-8', 'us-east1-b', 'projects/p/reservations/g',
              3, targeted=True)]


def test_nothing_counts_without_reservation_config():
    reservations.set_reservations(_inventory())
    assert not reservations.need_to_query()
    assert reservations.snapshot() is None
    assert reservations.available('aws', 'p3.2xlarge', 'us-west-2',
                                  'us-west-2b', False) == 0


def test_consumption_rules_follow_the_reference():
    reservations.set_reservations(_inventory())
    skypilot_config.set_config({'aws': {'prioritize_reservations': True}})
    avail = reservations.available
    # one count per name, the last listing wins (a dict in the reference);
    # the targeted one is not named
    assert avail('aws', 'p3.2xlarge', 'us-west-2', 'us-west-2b', False) == 2
    assert avail('aws', 'p3.2xlarge', 'us-west-2', 'us-west-2b', True) == 0
    assert avail('aws', 'p3.2xlarge', 'us-west-2', None, False) == 0
    assert avail('aws', 'p3.2xlarge', 'us-west-2', 'us-west-2a', False) == 0
    # GCP's listing is empty unless GCP's own config enables it
    assert avail('gcp', 'n1-highmem-8', 'us-east1', 'us-east1-b', False) == 0
    skypilot_config.set_config({
        'aws': {'specific_reservations': ['tgt']},
        'gcp': {'specific_reservations': ['projects/p/reservations/g']}})
    assert avail('aws', 'p3.2xlarge', 'us-west-2', 'us-west-2b', False) == 10
    assert avail('gcp', 'n1-highmem-8', 'us-east1', 'us-east1-b', False) == 3
    # clouds without reservations
    assert avail('azure', 'p3.2xlarge', 'eastus', 'us-west-2b', False) == 0


def test_specific_reservations_resolve_per_region_like_the_reference():
    """config_utils.get_cloud_config_value_from_dict: a region_configs
    override only exists for Nebius and OCI; AWS and GCP read the cloud
    level in every region."""
    skypilot_config.set_config({
        'aws': {'specific_reservations': ['a'],
                'region_configs': {'us-west-2': {'specific_reservations':
                                                 ['b']}}},
        'oci': {'specific_reservations': ['a'],
                'region_configs': {'us-ashburn-1': {'specific_reservations':
                                                    ['b']}}}})
    assert reservations.specific_reservations('aws', 'us-west-2') == {'a'}
    assert reservations.specific_reservations('oci', 'us-ashburn-1') == {'b'}
    assert reservations.specific_reservations('oci', 'us-phoenix-1') == {'a'}
    assert reservations.specific_reservations('oci', None) == {'a'}


def test_provider_is_called_for_the_inventory():
    calls = []

    def provider():
        calls.append(1)
        return [dict(cloud='aws', instance_type='p3.2xlarge',
                     zone='us-west-2b', name='x', available=5)]

    reservations.set_provider(provider)
    skypilot_config.set_config({'aws': {'prioritize_reservations': True}})
    assert reservations.available('aws', 'p3.2xlarge', 'us-west-2',
                                  'us-west-2b', False) == 5
    assert calls
    # an explicit inventory takes precedence
    reservations.set_reservations([])
    assert reservations.available('aws', 'p3.2xlarge', 'us-west-2',
                                  'us-west-2b', False) == 0


def test_aws_optimize_by_zone_follows_the_config():
    assert not aws_lib.AWS.optimize_by_zone()
    for cfg in ({'aws': {'prioritize_reservations': True}},
                {'aws': {'specific_reservations': ['r']}}):
        skypilot_config.set_config(cfg)
        assert aws_lib.AWS.optimize_by_zone()
    for cfg in ({'aws': {'specific_reservations': []}},
                {'aws': {'prioritize_reservations': False}},
                {'gcp': {'prioritize_reservations': True}}):
        skypilot_config.set_config(cfg)
        assert not aws_lib.AWS.optimize_by_zone()
    assert gcp_lib.GCP.optimize_by_zone()


def test_device_table_sums_consumable_counts_per_key():
    store = runner.activate_catalog(reservation_scenarios.CATALOG)
    skypilot_config.set_config({'aws': {'prioritize_reservations': True},
                                'gcp': {'prioritize_reservations': True}})
    reservations.set_reservations(
        reservation_scenarios.RESERVATION_INVENTORY +
        [dict(cloud='aws', instance_type='no-such-type', zone='us-west-2b',
              name='x', available=1),
         dict(cloud='aws', instance_type='p3.2xlarge', zone='nowhere-1a',
              name='y', available=1)])
    table = reservations.device_table(store, reservations.snapshot())
    assert table.dtype == _native.RESERVATION_DTYPE
    keys = [tuple(int(v) for v in r)[:3] for r in table]
    assert keys == sorted(set(keys))
    aws = store.cloud('aws')
    gcp = store.cloud('gcp')
    got = {(int(r['cloud']), int(r['inst_id']), int(r['zone_id'])):
           int(r['count']) for r in table}
    want = {
        (aws.index, aws.inst_index['p3.2xlarge'],
         aws.zone_exact['us-west-2b']): 4,
        # the targeted cr-tgt-w2c and g-req are not named: left out
        (aws.index, aws.inst_index['p3.2xlarge'],
         aws.zone_exact['us-east-2a']): 0,
        (aws.index, aws.inst_index['m6i.2xlarge'],
         aws.zone_exact['us-east-2b']): 2,
        (gcp.index, gcp.inst_index['n1-highmem-8'],
         gcp.zone_exact['us-east1-b']): 3,
        (gcp.index, gcp.inst_index['n1-standard-8'],
         gcp.zone_exact['us-east1-b']): 3,
        (gcp.index, gcp.inst_index['a2-highgpu-1g'],
         gcp.zone_exact['us-east4-a']): 2,
    }
    assert got == want


def test_reservation_record_layout():
    assert _native.ABI_VERSION == 4
    assert _native.SLOT_DTYPE.itemsize == 80
    assert _native.SLOT_DTYPE.fields['pad_'][1] == 52
    assert _native.RESERVATION_DTYPE.itemsize == 16
    assert [_native.RESERVATION_DTYPE.fields[n][1] for n in
            ('cloud', 'inst_id', 'zone_id', 'count')] == [0, 4, 8, 12]
    names = [n for n, _ in _native.Problem._fields_]  # pylint: disable=protected-access
    assert names[-2:] == ['reservations', 'n_reservations']
    assert np.zeros(1, _native.RESERVATION_DTYPE).nbytes == 16
