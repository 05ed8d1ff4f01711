"""Regenerate tests/golden/cost_report.json from the UNMODIFIED reference.

Build container only (needs the reference tree, see bootstrap.py):

    python oracle/ref_harness/gen_cost_report.py

Each record is a cluster-history entry as sky.core.cost_report sees it
(sky/core.py:446-468): name, duration, num_nodes and the launched Resources,
whose cloud, instance type, accelerators, spot flag, region and zone are set
as a launched cluster's pickled Resources carries them (no validation: a type
or zone may have left the catalog since). The records are drawn, seeded, from
the catalogs themselves: on-demand and spot, with no region, a region or a
zone, GCP hosts with attached accelerators and TPU VMs, vSphere (every
instance free), an unknown instance type, a zone without the type, a region
that does not exist, a zone on a cloud without zones, accelerators GCP does
not offer and types without any spot price. The reference computes
`get_cost(duration) * num_nodes` for each, or the warning it logs when that
raises. The AWS catalog of tests/azmap_scenarios.py carries zone IDs and the
reference maps them to zone names through the account's az_mappings file.
Records where the reference's spot -> on-demand fallback for GCP accelerators
meets pandas' all-NA idxmin error are flagged `pandas_all_na`, with the total
the fallback intends (`fallback_total`): the reference's instance price plus
its on-demand accelerator price for the same region and zone. One record per
catalog has no Resources at all, as a history record whose launched resources
could not be restored.
"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pandas as pd

_HERE = os.path.dirname(os.path.abspath(__file__))
_REPO = os.path.dirname(os.path.dirname(_HERE))
sys.path.insert(0, _REPO)
sys.path.insert(0, _HERE)

_IDENTITY = 'AIDAEXAMPLEUSERID0001'


def catalogs():
    from tests import azmap_scenarios  # pylint: disable=import-outside-toplevel
    from tests import scenarios  # pylint: disable=import-outside-toplevel
    out = {name: dict(scenarios.CATALOGS[name])
           for name in ('multi6k', 'gpuclouds', 'three4k', 'vsphere3k')}
    out['azmap'] = dict(azmap_scenarios.CATALOG)
    return out


def _rec(out, rng, name, cloud, instance_type, accelerators=None,
         use_spot=False, region=None, zone=None):
    out.append({
        'name': name, 'duration': int(rng.integers(60, 3_000_000)),
        'num_nodes': int(rng.integers(1, 5)), 'cloud': cloud,
        'instance_type': instance_type, 'accelerators': accelerators,
        'use_spot': use_spot, 'region': region, 'zone': zone
    })


def make_records(cat_name, frames, seed):
    """Seeded records over the catalog `frames` (zone names as the user
    sees them)."""
    rng = np.random.default_rng(seed)
    out = []
    for cloud, df in frames.items():
        insts = df[df['InstanceType'].notna()]
        types = sorted(insts['InstanceType'].unique())
        has_zone_col = 'AvailabilityZone' in df.columns
        pick = rng.choice(types, size=min(6, len(types)), replace=False)
        for j, it in enumerate(pick):
            rows = insts[insts['InstanceType'] == it]
            row = rows.iloc[int(rng.integers(len(rows)))]
            zone = row['AvailabilityZone'] if has_zone_col else None
            places = [(None, None), (row['Region'], None)]
            if zone is not None and not pd.isna(zone):
                places.append((row['Region'], zone))
            for spot in (False, True):
                for k, (rg, zn) in enumerate(places):
                    _rec(out, rng, f'{cat_name}-{cloud}-{j}-{int(spot)}{k}',
                         cloud, str(it), None, spot, rg, zn)
        # a type without any spot price, asked for spot
        no_spot = insts.groupby('InstanceType')['SpotPrice'].apply(
            lambda s: s.isna().all())
        for it in sorted(no_spot[no_spot].index)[:2]:
            _rec(out, rng, f'{cat_name}-{cloud}-nospot-{it}', cloud, str(it),
                 None, True)
        # a zone of the cloud without rows of the type
        if has_zone_col:
            it = str(pick[0])
            have = set(insts[insts['InstanceType'] == it]
                       ['AvailabilityZone'].dropna())
            others = sorted(set(df['AvailabilityZone'].dropna()) - have)
            if others:
                _rec(out, rng, f'{cat_name}-{cloud}-otherzone', cloud, it,
                     None, False, None, others[0])
        else:
            _rec(out, rng, f'{cat_name}-{cloud}-zoneless', cloud,
                 str(pick[0]), None, False, None, 'zone-a')
        _rec(out, rng, f'{cat_name}-{cloud}-unknown', cloud,
             'no-such-type.large')
        _rec(out, rng, f'{cat_name}-{cloud}-noregion', cloud, str(pick[0]),
             None, False, 'nowhere-1')
    if 'gcp' in frames:
        df = frames['gcp']
        accs = df[df['InstanceType'].isna() & df['AcceleratorName'].notna()]
        hosts = sorted(t for t in df['InstanceType'].dropna().unique()
                       if str(t).startswith('n1-'))
        for j in range(min(12, len(accs))):
            row = accs.iloc[int(rng.integers(len(accs)))]
            name = str(row['AcceleratorName'])
            count = float(row['AcceleratorCount'])
            acc = {name: int(count) if count.is_integer() else count}
            host = ('TPU-VM' if name.startswith('tpu-') and j % 2 == 0 else
                    str(hosts[int(rng.integers(len(hosts)))]))
            for spot in (False, True):
                for k, (rg, zn) in enumerate(
                    [(None, None), (row['Region'], None),
                     (row['Region'], row['AvailabilityZone'])]):
                    _rec(out, rng, f'{cat_name}-gcpacc-{j}-{int(spot)}{k}',
                         'gcp', host, acc, spot, rg, zn)
        if hosts:
            for k, rg in enumerate((None, 'us-central1')):
                _rec(out, rng, f'{cat_name}-gcpacc-missing-{k}', 'gcp',
                     str(hosts[0]), {'V100': 3}, False, rg)
    # a record whose launched resources could not be restored
    # (global_user_state.get_clusters_from_history gives None)
    _rec(out, rng, f'{cat_name}-no-resources', None, None)
    out[-1]['resources_none'] = True
    return out


def _launched(sky, spec):
    """The launched Resources of a record, as the cluster table restores it:
    fields set as they were at launch; None where it could not be
    restored."""
    from sky.utils import registry  # pylint: disable=import-outside-toplevel
    if spec.get('resources_none'):
        return None
    r = sky.Resources(cloud=registry.CLOUD_REGISTRY.from_str(spec['cloud']))
    # pylint: disable=protected-access
    r._instance_type = spec['instance_type']
    r._accelerators = spec['accelerators']
    r._use_spot = spec['use_spot']
    r._region = spec['region']
    r._zone = spec['zone']
    return r


def _fallback_total(sky, spec):
    """get_cost's total with the accelerators priced on demand: what
    get_accelerator_hourly_cost returns when no row has a spot price
    (gcp_catalog.py:433-439), computed by the reference's own functions."""
    from sky.catalog import gcp_catalog  # pylint: disable=import-outside-toplevel
    r = _launched(sky, spec)
    hourly = r.cloud.instance_type_to_hourly_cost(r.instance_type, r.use_spot,
                                                  r.region, r.zone)
    (acc, count), = r.accelerators.items()
    hourly += gcp_catalog.get_accelerator_hourly_cost(
        acc, count, use_spot=False, region=r.region, zone=r.zone)
    return float(hourly * (spec['duration'] / 3600)) * spec['num_nodes']


def _run_child(cat_name, spec_json, out_path):
    import bootstrap  # pylint: disable=import-outside-toplevel
    from skypilot_b200 import synth  # pylint: disable=import-outside-toplevel
    spec = json.loads(spec_json)
    frames = synth.make_catalogs(**spec)
    mapping = None
    if spec.get('aws_zone_ids'):
        from tests import azmap_scenarios  # pylint: disable=import-outside-toplevel
        _, mapping = azmap_scenarios.frames_and_mapping()
    from skypilot_b200.catalog import store as store_lib  # pylint: disable=import-outside-toplevel
    named = dict(frames)
    if mapping is not None:
        named['aws'] = store_lib.apply_az_mapping(frames['aws'], mapping)
    records = make_records(cat_name, named, seed=len(cat_name) * 1009)
    with tempfile.TemporaryDirectory(prefix='skyref_home_') as home:
        bootstrap.write_catalogs(home, frames)
        if mapping is not None:
            aws_dir = os.path.join(home, '.sky', 'catalogs', 'v8', 'aws')
            digest = hashlib.md5(_IDENTITY.encode()).hexdigest()[:8]
            mapping.to_csv(os.path.join(aws_dir, f'az_mappings-{digest}.csv'),
                           index=False)
        sky = bootstrap.import_reference(home, list(frames))
        if mapping is not None:
            from sky.clouds import aws  # pylint: disable=import-outside-toplevel
            aws.AWS.get_active_user_identity = classmethod(
                lambda cls: [_IDENTITY])
        for rec in records:
            try:
                launched = _launched(sky, rec)
                rec['total_cost'] = (launched.get_cost(rec['duration']) *
                                     rec['num_nodes'])
                rec['failed'] = False
            except Exception as e:  # pylint: disable=broad-except
                rec['total_cost'] = 0.0
                rec['failed'] = True
                rec['warning'] = (f'Failed to get total cost for cluster '
                                  f'{rec["name"]}: {str(e)}')
                # pandas >= 3 raises on Series.idxmin over all-NA values,
                # where earlier versions returned NaN and
                # get_accelerator_hourly_cost falls back to the on-demand
                # price (gcp_catalog.py:437-439)
                rec['pandas_all_na'] = 'Encountered all NA values' in str(e)
                if rec['pandas_all_na']:
                    rec['fallback_total'] = _fallback_total(sky, rec)
    with open(out_path, 'w', encoding='utf-8') as f:
        json.dump(records, f)


def main():
    ref = os.path.join(_REPO, 'oracle', '_ref')
    if 'SKYOPT_REFERENCE_ROOT' not in os.environ and os.path.isdir(
            os.path.join(ref, 'sky')):
        os.environ['SKYOPT_REFERENCE_ROOT'] = ref  # what build() copied
    payload = {
        'generated_by': 'oracle/ref_harness/gen_cost_report.py',
        'reference': 'skypilot-org/skypilot @ 7808630 (unmodified)',
        'catalogs': {}
    }
    for cat_name, spec in catalogs().items():
        tmp_out = os.path.join(tempfile.gettempdir(),
                               f'cost_report_{cat_name}_{os.getpid()}.json')
        cmd = [sys.executable, os.path.abspath(__file__), '--child', cat_name,
               json.dumps(spec), tmp_out]
        proc = subprocess.run(cmd, cwd='/tmp', check=False)
        if proc.returncode != 0:
            raise SystemExit(f'reference harness failed ({cat_name})')
        with open(tmp_out, encoding='utf-8') as f:
            records = json.load(f)
        os.unlink(tmp_out)
        payload['catalogs'][cat_name] = {'catalog': spec, 'records': records}
        print(f'[gen_cost_report] {cat_name}: {len(records)} records, '
              f'{sum(r["failed"] for r in records)} failed', flush=True)
    out_path = os.path.join(_REPO, 'tests', 'golden', 'cost_report.json')
    with open(out_path, 'w', encoding='utf-8') as f:
        json.dump(payload, f, separators=(',', ':'), sort_keys=True)
    print(f'[gen_cost_report] wrote {out_path}', flush=True)


if __name__ == '__main__':
    if '--child' in sys.argv:
        i = sys.argv.index('--child')
        _run_child(*sys.argv[i + 1:i + 4])
    else:
        main()
