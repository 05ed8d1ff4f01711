"""Regenerate tests/golden/reservations.json from the UNMODIFIED reference.

Build container only (needs the reference tree, see bootstrap.py):

    python oracle/ref_harness/gen_reservations.py

The scenarios are tests/reservation_scenarios.py. Each runs through
run_reference.py's `run_scenario` with the two calls that reach a cloud API
answered from the scenario's `reservations` inventory: the EC2 client behind
aws_utils.list_reservations_for_instance_type
(`describe_capacity_reservations`) and the `gcloud compute reservations list`
command behind gcp_utils' listing. Everything above those calls -- the config
gating, the consumption rules, the optimizer -- is the reference's own code.
The fixtures are committed; the GPU box never runs this script.
"""
import json
import os
import subprocess
import sys
import tempfile
import types

_HERE = os.path.dirname(os.path.abspath(__file__))
_REPO = os.path.dirname(os.path.dirname(_HERE))
sys.path.insert(0, _REPO)
sys.path.insert(0, _HERE)


class _FakeEc2:
    """`describe_capacity_reservations` over a seeded inventory."""

    def __init__(self, inventory):
        self.inventory = inventory

    def describe_capacity_reservations(self, Filters):  # pylint: disable=invalid-name
        inst = next(f['Values'][0] for f in Filters
                    if f['Name'] == 'instance-type')
        return {'CapacityReservations': [{
            'CapacityReservationId': r['name'], 'InstanceType': inst,
            'AvailabilityZone': r['zone'],
            'AvailableInstanceCount': r['available'],
            'InstanceMatchCriteria': 'targeted' if r.get('targeted') else
                                     'open',
        } for r in self.inventory
            if r['cloud'] == 'aws' and r['instance_type'] == inst]}


def _gcloud_listing(inventory, cmd):
    """stdout of `gcloud compute reservations list` (gcp_utils.py:131-171)."""
    inst = cmd.split('machineType=')[1].split(' ')[0]
    out = []
    for r in inventory:
        if r['cloud'] != 'gcp' or r['instance_type'] != inst:
            continue
        _, project, _, name = r['name'].split('/')
        zone = ('https://www.googleapis.com/compute/v1/projects/'
                f'{project}/zones/{r["zone"]}')
        out.append({'selfLink': f'{zone}/reservations/{name}', 'zone': zone,
                    'specificReservation': {'count': r['available'],
                                            'inUseCount': 0},
                    'specificReservationRequired': bool(r.get('targeted'))})
    return json.dumps(out)


def _run_child():
    """run_reference.py's main with the listings answered per scenario."""
    import run_reference  # pylint: disable=import-outside-toplevel
    original = run_reference.run_scenario

    def run_scenario(sky, scenario):
        if 'reservations' not in scenario or scenario.get('_in_reservations'):
            return original(sky, scenario)
        from sky.clouds.utils import aws_utils  # pylint: disable=import-outside-toplevel
        from sky.clouds.utils import gcp_utils  # pylint: disable=import-outside-toplevel
        inventory = scenario['reservations']
        listings = (aws_utils.list_reservations_for_instance_type,
                    gcp_utils._list_reservations_for_instance_type)  # pylint: disable=protected-access
        saved = (aws_utils.aws, gcp_utils.subprocess_utils)
        aws_utils.aws = types.SimpleNamespace(
            client=lambda *a, **k: _FakeEc2(inventory))
        real = gcp_utils.subprocess_utils
        fake = types.SimpleNamespace(**{
            k: getattr(real, k) for k in dir(real) if not k.startswith('__')})
        fake.run_with_retries = lambda cmd, **k: (
            0, _gcloud_listing(inventory, cmd), '')
        gcp_utils.subprocess_utils = fake
        for fn in listings:
            fn.cache_clear()
        try:
            return original(sky, dict(scenario, _in_reservations=True))
        finally:
            aws_utils.aws, gcp_utils.subprocess_utils = saved
            for fn in listings:
                fn.cache_clear()

    # run_reference's own recursion (per-scenario config) comes back here
    run_reference.run_scenario = run_scenario
    run_reference.main()


def main():
    from tests import reservation_scenarios  # pylint: disable=import-outside-toplevel
    spec = reservation_scenarios.CATALOG
    suite = reservation_scenarios.reservation_scenarios()
    with tempfile.NamedTemporaryFile('w', suffix='.json', delete=False) as f:
        json.dump(suite, f)
        sc_path = f.name
    out_path = os.path.join(_REPO, 'tests', 'golden', 'reservations.json')
    tmp_out = out_path + '.tmp'
    cmd = [sys.executable, os.path.abspath(__file__), '--child', '--catalog',
           json.dumps(spec), '--scenarios', sc_path, '--out', tmp_out]
    print('[gen_reservations]', len(suite), 'scenarios', flush=True)
    proc = subprocess.run(cmd, cwd='/tmp', stdout=subprocess.DEVNULL,
                          check=False)
    os.unlink(sc_path)
    if proc.returncode != 0:
        raise SystemExit('reference harness failed')
    with open(tmp_out, encoding='utf-8') as f:
        records = json.load(f)
    os.unlink(tmp_out)
    # compact candidates: [cloud, instance_type, region, zone, value]
    for rec in records:
        if 'candidates' in rec:
            rec['candidates'] = [[[
                c['cloud'], c['instance_type'], c['region'], c['zone'],
                c['value']
            ] for c in cands] for cands in rec['candidates']]
    payload = {
        'catalog': spec,
        'generated_by': 'oracle/ref_harness/gen_reservations.py',
        'reference': 'skypilot-org/skypilot @ 7808630 (unmodified)',
        'records': records
    }
    with open(out_path, 'w', encoding='utf-8') as f:
        json.dump(payload, f, separators=(',', ':'), sort_keys=True)
    n_err = sum('error' in r for r in records)
    print(f'[gen_reservations] wrote {out_path}: {len(records)} records, '
          f'{n_err} errors', flush=True)


if __name__ == '__main__':
    if '--child' in sys.argv:
        sys.argv.remove('--child')
        _run_child()
    else:
        main()
