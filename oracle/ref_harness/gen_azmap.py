"""Regenerate tests/golden/azmap.json and tests/golden/azmap_reservations.json
from the UNMODIFIED reference.

Build container only (needs the reference tree, see bootstrap.py):

    python oracle/ref_harness/gen_azmap.py

The scenarios are tests/azmap_scenarios.py. The scratch catalog directory
gets the AWS catalog with zone IDs and two `aws/az_mappings-*.csv` files: the
account's mapping (synth.aws_az_mapping) and a decoy made from another seed.
The reference chooses between them itself (sky/catalog/aws_catalog.py:
120-185), and runs twice:

  * identity: AWS.get_active_user_identity returns a fixed identity, the
    account's file is named by md5(identity)[:8] and is the OLDER file, so
    only the hash rule picks it;
  * newest: the identity call raises CloudUserIdentityError, the account's
    file is the NEWER one, so only the newest-file rule picks it.

Both runs must give the same records. Reservation scenarios go through
gen_reservations.py's inventory stubs. The fixtures are committed; the GPU
box never runs this script.
"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

_HERE = os.path.dirname(os.path.abspath(__file__))
_REPO = os.path.dirname(os.path.dirname(_HERE))
sys.path.insert(0, _REPO)
sys.path.insert(0, _HERE)

IDENTITY = 'AIDAEXAMPLEUSERID0001'


def _account_file(mode: str) -> str:
    if mode == 'identity':
        return f'az_mappings-{hashlib.md5(IDENTITY.encode()).hexdigest()[:8]}.csv'
    return 'az_mappings-newest00.csv'


def _run_child(mode: str, mapping_seed: int):
    import bootstrap  # pylint: disable=import-outside-toplevel
    import gen_reservations  # pylint: disable=import-outside-toplevel
    from skypilot_b200 import synth  # pylint: disable=import-outside-toplevel
    write_catalogs, import_reference = (bootstrap.write_catalogs,
                                        bootstrap.import_reference)

    def write_with_mappings(home, catalogs, *args, **kwargs):
        write_catalogs(home, catalogs, *args, **kwargs)
        aws_dir = os.path.join(home, '.sky', 'catalogs', 'v8', 'aws')
        account = os.path.join(aws_dir, _account_file(mode))
        decoy = os.path.join(aws_dir, 'az_mappings-decoy000.csv')
        synth.aws_az_mapping(catalogs['aws'], mapping_seed).to_csv(
            account, index=False)
        synth.aws_az_mapping(catalogs['aws'], mapping_seed + 1).to_csv(
            decoy, index=False)
        older, newer = (account, decoy) if mode == 'identity' else (decoy,
                                                                   account)
        os.utime(older, (1_600_000_000, 1_600_000_000))
        os.utime(newer, (1_700_000_000, 1_700_000_000))

    def import_with_identity(home, enabled):
        sky = import_reference(home, enabled)
        from sky import exceptions  # pylint: disable=import-outside-toplevel
        from sky.clouds import aws  # pylint: disable=import-outside-toplevel

        def identity(cls):
            del cls
            if mode == 'identity':
                return [IDENTITY]
            raise exceptions.CloudUserIdentityError('no AWS credentials')

        aws.AWS.get_active_user_identity = classmethod(identity)
        return sky

    bootstrap.write_catalogs = write_with_mappings
    bootstrap.import_reference = import_with_identity
    gen_reservations._run_child()  # pylint: disable=protected-access


def _compact(records):
    # compact candidates: [cloud, instance_type, region, zone, value]
    for rec in records:
        if 'candidates' in rec:
            rec['candidates'] = [[[
                c['cloud'], c['instance_type'], c['region'], c['zone'],
                c['value']
            ] for c in cands] for cands in rec['candidates']]
    return records


def _order_differs_under_ids(records, mapping):
    """Records with a candidate table whose order changes when zone names
    are replaced by their IDs: ties at equal value inside a region are
    ordered by zone (common.py:797-802)."""
    to_id = dict(zip(mapping['AvailabilityZoneName'],
                     mapping['AvailabilityZone']))
    out = []
    for rec in records:
        for cands in rec.get('candidates', []):
            zoned = [c for c in cands if c[0] == 'aws' and c[3] is not None]
            key_names = [(c[4], c[2], c[3]) for c in zoned]
            key_ids = [(c[4], c[2], to_id[c[3]]) for c in zoned]
            by_names = sorted(range(len(zoned)), key=key_names.__getitem__)
            by_ids = sorted(range(len(zoned)), key=key_ids.__getitem__)
            if by_names != by_ids:
                out.append(rec['name'])
                break
    return out


def main():
    from tests import azmap_scenarios  # pylint: disable=import-outside-toplevel
    spec = azmap_scenarios.CATALOG
    plain = (azmap_scenarios.azmap_scenarios() +
             azmap_scenarios.listing_cases() +
             azmap_scenarios.job_group_cases())
    resv = azmap_scenarios.reservation_scenarios()
    suite = plain + resv
    with tempfile.NamedTemporaryFile('w', suffix='.json', delete=False) as f:
        json.dump(suite, f)
        sc_path = f.name
    runs = {}
    for mode in ('identity', 'newest'):
        tmp_out = os.path.join(tempfile.gettempdir(),
                               f'azmap_{mode}_{os.getpid()}.json')
        cmd = [sys.executable, os.path.abspath(__file__), '--child', mode,
               str(azmap_scenarios.AZ_MAPPING_SEED), '--catalog',
               json.dumps(spec), '--scenarios', sc_path, '--out', tmp_out]
        print('[gen_azmap]', mode, len(suite), 'scenarios', flush=True)
        proc = subprocess.run(cmd, cwd='/tmp', stdout=subprocess.DEVNULL,
                              check=False)
        if proc.returncode != 0:
            raise SystemExit(f'reference harness failed ({mode})')
        with open(tmp_out, encoding='utf-8') as f:
            runs[mode] = _compact(json.load(f))
        os.unlink(tmp_out)
    os.unlink(sc_path)
    def decided(records):
        # with several common infras the reference's JobGroup pick is the
        # first element of a set: it may differ from run to run
        return [{k: v for k, v in r.items()
                 if len(r.get('common_infras', [])) < 2 or
                 k not in ('plan', 'overrides')} for r in records]

    if decided(runs['identity']) != decided(runs['newest']):
        differ = [a['name'] for a, b in zip(runs['identity'], runs['newest'])
                  if a != b]
        raise SystemExit(f'the two ways of choosing the mapping differ: '
                         f'{differ}')
    records = runs['identity']
    resv_names = {s['name'] for s in resv}
    _, mapping = azmap_scenarios.frames_and_mapping()
    for name, part in (('azmap', [r for r in records
                                  if r['name'] not in resv_names]),
                       ('azmap_reservations',
                        [r for r in records if r['name'] in resv_names])):
        payload = {
            'catalog': spec,
            'az_mapping_seed': azmap_scenarios.AZ_MAPPING_SEED,
            'generated_by': 'oracle/ref_harness/gen_azmap.py',
            'reference': 'skypilot-org/skypilot @ 7808630 (unmodified)',
            'records': part
        }
        out_path = os.path.join(_REPO, 'tests', 'golden', f'{name}.json')
        with open(out_path, 'w', encoding='utf-8') as f:
            json.dump(payload, f, separators=(',', ':'), sort_keys=True)
        n_err = sum('error' in r for r in part)
        print(f'[gen_azmap] wrote {out_path}: {len(part)} records, '
              f'{n_err} errors', flush=True)
    differs = _order_differs_under_ids(records, mapping)
    print(f'[gen_azmap] {len(differs)} records order AWS zones differently '
          f'under zone IDs: {differs}', flush=True)


if __name__ == '__main__':
    if '--child' in sys.argv:
        i = sys.argv.index('--child')
        mode, seed = sys.argv[i + 1], int(sys.argv[i + 2])
        del sys.argv[i:i + 3]
        _run_child(mode, seed)
    else:
        main()
