"""Capacity-reservation scenarios (skypilot_b200/reservations.py) in the
schema of tests/scenarios.py, plus two keys:

  reservations  the inventory the reference's cloud listings return
                (aws_utils.list_reservations_for_instance_type, gcp_utils'
                gcloud listing), as skypilot_b200.reservations records; GCP
                names are the ones the reference derives from a selfLink
                ('projects/<p>/reservations/<r>')
  config        the SkyPilot config that turns them on

oracle/ref_harness/gen_reservations.py runs them through the unmodified
reference (tests/golden/reservations.json)."""
import copy

from tests import scenarios

CATALOG = dict(scenarios.CATALOGS['multi6k'])

_single = scenarios._single  # pylint: disable=protected-access
_chain = scenarios._chain  # pylint: disable=protected-access
_job_group = scenarios._job_group  # pylint: disable=protected-access

RESERVATION_INVENTORY = [
    dict(cloud='aws', instance_type='p3.2xlarge', zone='us-west-2b',
         name='cr-open-w2b', available=4),
    dict(cloud='aws', instance_type='p3.2xlarge', zone='us-west-2c',
         name='cr-tgt-w2c', available=8, targeted=True),
    dict(cloud='aws', instance_type='p3.2xlarge', zone='us-east-2a',
         name='cr-zero', available=0),
    dict(cloud='aws', instance_type='m6i.2xlarge', zone='us-east-2b',
         name='cr-cpu', available=1),
    dict(cloud='aws', instance_type='m6i.2xlarge', zone='us-east-2b',
         name='cr-cpu-2', available=1),
    dict(cloud='gcp', instance_type='n1-highmem-8', zone='us-east1-b',
         name='projects/p/reservations/g-open', available=3),
    dict(cloud='gcp', instance_type='n1-standard-8', zone='us-east1-b',
         name='projects/p/reservations/g-open8', available=3),
    dict(cloud='gcp', instance_type='n1-highmem-8', zone='us-west1-b',
         name='projects/p/reservations/g-req', available=8, targeted=True),
    dict(cloud='gcp', instance_type='a2-highgpu-1g', zone='us-east4-a',
         name='projects/p/reservations/a2', available=2),
]

_AWS_PRIO = {'aws': {'prioritize_reservations': True}}
_GCP_PRIO = {'gcp': {'prioritize_reservations': True}}
_BOTH_PRIO = {'aws': {'prioritize_reservations': True},
              'gcp': {'prioritize_reservations': True}}


def reservation_scenarios():
    """Reservations on the multi6k catalog: plans a reservation flips,
    partial coverage, consumption rules, spot, a chain with egress, a
    diamond, a blocked list, TIME, an empty inventory and a JobGroup."""

    def resv(s, config, inventory=None):
        s['config'] = config
        s['reservations'] = copy.deepcopy(
            RESERVATION_INVENTORY if inventory is None else inventory)
        return s

    s = [
        resv(_single('aws_prio_v100_n4', accelerators='V100', num_nodes=4),
             _AWS_PRIO),
        resv(_single('aws_prio_v100_n6_partial', accelerators='V100',
                     num_nodes=6), _AWS_PRIO),
        resv(_single('aws_prio_v100_n8_targeted_unnamed', accelerators='V100',
                     num_nodes=8), _AWS_PRIO),
        resv(_single('aws_specific_v100_n8', accelerators='V100', num_nodes=8),
             {'aws': {'specific_reservations': ['cr-tgt-w2c']}}),
        # the reference reads region_configs for Nebius / OCI only
        resv(_single('aws_region_override_v100_n8', accelerators='V100',
                     num_nodes=8),
             {'aws': {'prioritize_reservations': True, 'region_configs': {
                 'us-west-2': {'specific_reservations': ['cr-tgt-w2c']}}}}),
        resv(_single('aws_prio_cpu_n2', cloud='aws', cpus='8+', num_nodes=2),
             _AWS_PRIO),
        resv(_single('aws_prio_spot_v100_n4', accelerators='V100', num_nodes=4,
                     use_spot=True), _AWS_PRIO),
        resv(_single('gcp_prio_v100_n3', cloud='gcp', accelerators='V100',
                     num_nodes=3), _GCP_PRIO),
        resv(_single('gcp_prio_v100_n8_required_unnamed', cloud='gcp',
                     accelerators='V100', num_nodes=8), _GCP_PRIO),
        resv(_single('gcp_specific_v100_n8', cloud='gcp', accelerators='V100',
                     num_nodes=8),
             {'gcp': {'specific_reservations':
                      ['projects/p/reservations/g-req']}}),
        resv(_single('gcp_prio_a100_n2', cloud='gcp', accelerators='A100',
                     num_nodes=2), _GCP_PRIO),
        # GCP's config alone: AWS records do not count, AWS is not split
        resv(_single('gcp_only_config_v100_n4', accelerators='V100',
                     num_nodes=4), _GCP_PRIO),
        resv(_single('both_prio_v100_n5', accelerators='V100', num_nodes=5),
             _BOTH_PRIO),
        resv(_single('aws_prio_empty_inventory_v100', accelerators='V100'),
             _AWS_PRIO, inventory=[]),
        resv(_single('aws_prio_empty_inventory_cpu_n2', cpus='8+',
                     num_nodes=2), _AWS_PRIO, inventory=[]),
    ]
    time = resv(_single('aws_prio_v100_n4_time', accelerators='V100',
                        num_nodes=4), _AWS_PRIO)
    time['minimize'] = 'time'
    time['tasks'][0]['time_est'] = {'default': 7200, 'by_cloud': {'gcp': 3600}}
    s.append(time)
    blocked = resv(_single('aws_prio_v100_n4_blocked', accelerators='V100',
                           num_nodes=4), _AWS_PRIO)
    blocked['blocked'] = [{'cloud': 'aws', 'zone': 'us-west-2b'}]
    s.append(blocked)
    s.append(resv(_chain('chain3_egress', [
        {'accelerators': 'V100', 'num_nodes': 4, 'outputs_gb': 100},
        {'cpus': '8+', 'num_nodes': 2, 'outputs_gb': 20},
        {'accelerators': 'V100', 'num_nodes': 3},
    ]), _BOTH_PRIO))
    diamond = resv(_chain('diamond4', [
        {'accelerators': 'V100', 'num_nodes': 4, 'outputs_gb': 10},
        {'cpus': '8+', 'num_nodes': 2, 'outputs_gb': 5},
        {'accelerators': 'A100', 'num_nodes': 2, 'outputs_gb': 5},
        {'accelerators': 'V100', 'num_nodes': 3},
    ]), _BOTH_PRIO)
    diamond['edges'] = [[0, 1], [0, 2], [1, 3], [2, 3]]
    s.append(diamond)
    s.append(resv(_job_group('jg_prio_two', [
        dict(accelerators='V100', num_nodes=4), dict(cpus='8+', num_nodes=2)
    ]), _BOTH_PRIO))
    return s
