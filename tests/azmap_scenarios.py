"""Scenarios on a catalog whose AWS zones are zone IDs, with an account's
zone mapping applied (skypilot_b200.catalog.store.apply_az_mapping), in the
schema of tests/scenarios.py.

CATALOG is the `azmap` catalog: AWS (zone IDs, `use1-az3`), GCP and RunPod.
AZ_MAPPING_SEED seeds synth.aws_az_mapping: per region the zone letters are a
permutation of the ID numbers, eu-north-1 and eu-west-2 are not mapped (the
account lacks them) and ap-east-1, ap-northeast-2 and me-south-1 lose one
zone. `reservations` / `config` keys are the ones of
tests/reservation_scenarios.py; AWS reservations carry zone names, as
describe_capacity_reservations reports them.

oracle/ref_harness/gen_azmap.py runs them through the unmodified reference
(tests/golden/azmap.json, tests/golden/azmap_reservations.json)."""
import copy

from skypilot_b200 import synth
from tests import scenarios

CATALOG = {'seed': 73, 'n_rows': 6000, 'clouds': ['aws', 'gcp', 'runpod'],
           'aws_zone_ids': True}
AZ_MAPPING_SEED = 73
# regions of the AWS catalog that the mapping drops entirely
UNMAPPED_REGIONS = ('eu-north-1', 'eu-west-2')

_single = scenarios._single  # pylint: disable=protected-access
_chain = scenarios._chain  # pylint: disable=protected-access
_job_group = scenarios._job_group  # pylint: disable=protected-access


def frames_and_mapping():
    """The catalog frames (zone IDs) and the account's mapping."""
    spec = dict(CATALOG)
    frames = synth.make_catalogs(**spec)
    return frames, synth.aws_az_mapping(frames['aws'], AZ_MAPPING_SEED)


def azmap_scenarios():
    """Placement on the mapped catalog: single tasks, spot (per-zone
    candidates), requests by zone name, by zone ID and by an unmapped region,
    blocked zones by name, chains and a diamond with egress, TIME, listings
    and a JobGroup."""
    s = [
        _single('v100', accelerators='V100'),
        _single('t4', accelerators='T4'),
        _single('a100x8', accelerators='A100:8'),
        _single('cpu_default'),
        _single('cpu_8p', cpus='8+'),
        _single('aws_cpu', cloud='aws', cpus='4+'),
        _single('aws_inst', cloud='aws', instance_type='p3.2xlarge'),
        _single('spot_v100', accelerators='V100', use_spot=True),
        _single('spot_aws_t4', cloud='aws', accelerators='T4', use_spot=True),
        _single('spot_aws_cpu', cloud='aws', cpus='8+', use_spot=True),
        _single('spot_aws_inst', cloud='aws', instance_type='g4dn.xlarge',
                use_spot=True),
        _single('spot_region_partly_mapped', cloud='aws',
                region='ap-northeast-2', cpus='4+', use_spot=True),
        _single('zone_name', infra='aws/us-east-1/us-east-1a',
                accelerators='V100'),
        _single('zone_name_spot', infra='aws/us-west-1/us-west-1d',
                cpus='4+', use_spot=True),
        _single('zone_id_rejected', infra='aws/us-east-1/use1-az3',
                accelerators='V100'),
        _single('unmapped_region', infra='aws/eu-west-2', cpus='4+'),
        _single('unmapped_region_spot', infra='aws/eu-north-1',
                accelerators='T4', use_spot=True),
        _single('mapped_region', infra='aws/eu-west-3', cpus='4+'),
        dict(_single('blocked_zones', cloud='aws', accelerators='T4',
                     use_spot=True),
             blocked=[{'cloud': 'aws', 'zone': 'us-east-1b'},
                      {'cloud': 'aws', 'zone': 'us-east-1e'},
                      {'cloud': 'aws', 'region': 'us-east-2'}]),
        dict(_single('blocked_zone_spot_cpu', cloud='aws', cpus='8+',
                     use_spot=True),
             blocked=[{'cloud': 'aws', 'zone': 'us-west-2c'}]),
        _chain('chain3_egress', [
            {'accelerators': 'V100', 'outputs_gb': 100},
            {'cloud': 'aws', 'cpus': '8+', 'use_spot': True,
             'outputs_gb': 20},
            {'accelerators': 'T4'}]),
        _chain('chain2_spot_egress', [
            {'accelerators': 'T4', 'use_spot': True, 'outputs_gb': 500},
            {'cpus': '8+', 'use_spot': True}]),
        _chain('chain8_cfg2', scenarios.CFG2_TASKS),
        _chain('chain2_time', [
            {'accelerators': 'V100', 'outputs_gb': 50,
             'time_est': {'default': 7200, 'by_acc': {'V100': 3000}}},
            {'cpus': '8+', 'use_spot': True, 'time_est': {'default': 600}}],
               minimize='time'),
    ]
    diamond = {
        'name': 'diamond_egress',
        'tasks': [
            {'name': 'a', 'resources': [{'accelerators': 'V100'}],
             'outputs_gb': 100},
            {'name': 'b', 'resources': [{'accelerators': 'T4',
                                         'use_spot': True}],
             'outputs_gb': 5},
            {'name': 'c', 'resources': [{'cpus': '32+', 'memory': '128+'}],
             'outputs_gb': 5},
            {'name': 'd', 'resources': [{'accelerators': 'A100:8'}]},
        ],
        'edges': [[0, 1], [0, 2], [1, 3], [2, 3]],
    }
    s.append(diamond)
    tdiam = copy.deepcopy(diamond)
    tdiam['name'] = 'diamond_time'
    tdiam['minimize'] = 'time'
    for i, secs in enumerate([3600, 1800, 7200, 900]):
        tdiam['tasks'][i]['time_est'] = {'default': secs}
    s.append(tdiam)
    return s


def listing_cases():
    def listing(name, **kwargs):
        return {'name': name, 'kind': 'list_accelerators', 'kwargs': kwargs}

    return [
        listing('aws_all', clouds=['aws']),
        listing('aws_all_regions', clouds=['aws'], all_regions=True),
        listing('aws_eu', clouds=['aws'], region_filter='eu-',
                all_regions=True),
        listing('aws_unmapped_region', clouds=['aws'],
                region_filter='eu-west-2', all_regions=True),
        listing('aws_gcp_region_east', clouds=['aws', 'gcp'],
                region_filter='east', gpus_only=False),
    ]


def job_group_cases():
    return [
        _job_group('jg_two', [dict(accelerators='V100'),
                              dict(cpus='8+', num_nodes=2)]),
    ]


_AWS_PRIO = {'aws': {'prioritize_reservations': True}}

# zone names of the mapped catalog (us-west-2b is usw2-az3, us-east-1a is
# use1-az3)
RESERVATION_INVENTORY = [
    dict(cloud='aws', instance_type='p3.2xlarge', zone='us-west-2b',
         name='cr-w2b', available=4),
    dict(cloud='aws', instance_type='p3.2xlarge', zone='us-east-1a',
         name='cr-e1a', available=2),
    dict(cloud='aws', instance_type='m6i.2xlarge', zone='us-east-2b',
         name='cr-cpu', available=1),
    # a zone ID never matches a record of the mapped catalog
    dict(cloud='aws', instance_type='p3.2xlarge', zone='usw2-az1',
         name='cr-by-id', available=8),
]


def reservation_scenarios():
    """AWS reservations by zone name: on-demand candidates are per zone, so
    equal prices inside a region are ordered by zone name."""

    def resv(sc):
        sc['config'] = _AWS_PRIO
        sc['reservations'] = copy.deepcopy(RESERVATION_INVENTORY)
        return sc

    return [
        resv(_single('resv_v100_n4', accelerators='V100', num_nodes=4)),
        resv(_single('resv_v100_n8', cloud='aws', accelerators='V100',
                     num_nodes=8)),
        resv(_single('resv_cpu_n2', cloud='aws', cpus='8+', num_nodes=2)),
        resv(_single('resv_v100_zone', infra='aws/us-east-1/us-east-1a',
                     accelerators='V100', num_nodes=3)),
        resv(_chain('resv_chain2', [
            {'accelerators': 'V100', 'num_nodes': 4, 'outputs_gb': 50},
            {'cloud': 'aws', 'cpus': '8+', 'num_nodes': 2}])),
    ]
