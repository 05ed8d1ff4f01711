"""Records for the batch price path (skypilot_b200.catalog.get_costs /
skypilot_b200.cost_report): the launched Resources of the fixture records of
tests/golden/cost_report.json (oracle/ref_harness/gen_cost_report.py) and
seeded random records over a catalog."""
import json
from typing import Any, Dict, List, Optional

import numpy as np
import pandas as pd

import skypilot_b200 as sky
from skypilot_b200 import synth
from skypilot_b200.catalog.store import CatalogStore
from skypilot_b200.utils import registry
from tests import azmap_scenarios
from tests import scenario_runner as runner

_stores: Dict[str, CatalogStore] = {}


def activate(spec: Dict[str, Any]) -> CatalogStore:
    """Makes the catalog of `spec` the active one; the zone-ID AWS catalog of
    the azmap scenarios gets the account's zone mapping."""
    if not spec.get('aws_zone_ids'):
        return runner.activate_catalog(spec)
    key = json.dumps(spec, sort_keys=True)
    store = _stores.get(key)
    if store is None:
        frames, mapping = azmap_scenarios.frames_and_mapping()
        store = CatalogStore.from_frames(frames, aws_az_mapping=mapping)
        _stores[key] = store
    sky.catalog.set_store(store)
    sky.check.set_enabled_clouds(sky.check.ALL_CATALOG_CLOUDS)
    return store


def launched(spec: Dict[str, Any]) -> Optional[sky.Resources]:
    """A record's launched Resources with the fields set as they were at
    launch (no validation, as a restored cluster record has them); None for
    a record whose resources could not be restored."""
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


def history(specs: List[Dict[str, Any]]) -> List[Dict[str, Any]]:
    """Cluster-history records as get_clusters_from_history yields them."""
    return [{'name': s['name'], 'duration': s['duration'],
             'num_nodes': s['num_nodes'], 'resources': launched(s)}
            for s in specs]


def random_specs(frames: Dict[str, pd.DataFrame], n: int,
                 seed: int) -> List[Dict[str, Any]]:
    """`n` seeded records over `frames`: rows' types and places, spot or
    not, region and zone set or unset, GCP accelerators on n1 hosts and TPU
    VMs, and a share of records that cannot be priced (unknown types and
    regions, zones without the type, zones on clouds without zones,
    accelerators GCP does not offer)."""
    rng = np.random.default_rng(seed)
    pools = []
    for cloud, df in frames.items():
        inst = df[df['InstanceType'].notna()]
        zones = (inst['AvailabilityZone'] if 'AvailabilityZone' in df.columns
                 else pd.Series([None] * len(inst), index=inst.index))
        pools.append((cloud, inst['InstanceType'].to_numpy(),
                      inst['Region'].to_numpy(), zones.to_numpy()))
    gcp = frames.get('gcp')
    if gcp is not None:
        accs = gcp[gcp['InstanceType'].isna() & gcp['AcceleratorName'].notna()]
        hosts = sorted(t for t in gcp['InstanceType'].dropna().unique()
                       if str(t).startswith('n1-'))
    out = []
    for i in range(n):
        spec = {'name': f'c{i}', 'duration': int(rng.integers(1, 5_000_000)),
                'num_nodes': int(rng.integers(1, 9)), 'accelerators': None,
                'use_spot': bool(rng.integers(2)), 'region': None,
                'zone': None}
        kind = rng.random()
        if gcp is not None and kind < 0.2 and len(accs):
            row = accs.iloc[int(rng.integers(len(accs)))]
            count = float(row['AcceleratorCount'])
            name = str(row['AcceleratorName'])
            spec['cloud'] = 'gcp'
            spec['accelerators'] = {
                name: int(count) if count.is_integer() else count}
            spec['instance_type'] = ('TPU-VM' if name.startswith('tpu-') and
                                     rng.random() < 0.5 else
                                     str(hosts[int(rng.integers(len(hosts)))]))
            place = rng.integers(3)
            if place >= 1:
                spec['region'] = str(row['Region'])
            if place == 2:
                spec['zone'] = str(row['AvailabilityZone'])
        else:
            cloud, types, regions, zones = pools[int(rng.integers(len(pools)))]
            j = int(rng.integers(len(types)))
            spec['cloud'] = cloud
            spec['instance_type'] = str(types[j])
            place = rng.integers(3)
            if place >= 1:
                spec['region'] = str(regions[j])
            if place == 2 and zones[j] is not None and not pd.isna(zones[j]):
                spec['zone'] = str(zones[j])
        if kind > 0.96:
            # records the catalog cannot price
            bad = int(rng.integers(5))
            if bad == 0:
                spec['instance_type'] = 'no-such-type.large'
            elif bad == 1:
                spec['region'] = 'nowhere-1'
            elif bad == 2:
                spec['zone'] = 'nowhere-1a'
            elif bad == 3 and gcp is not None:
                spec['cloud'] = 'gcp'
                spec['instance_type'] = str(hosts[0])
                spec['accelerators'] = {'V100': 3}
            else:
                spec['zone'] = str(zones[j]) if spec['cloud'] != 'gcp' else (
                    'us-central1-a')
        out.append(spec)
    return out


def catalog_frames(spec: Dict[str, Any]) -> Dict[str, pd.DataFrame]:
    return synth.make_catalogs(**{k: v for k, v in spec.items()
                                  if k != 'enabled'})
