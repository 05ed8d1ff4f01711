"""The AWS account's zone mapping in the portable oracle.

Every AWS catalog function of the reference reads `_get_df()`
(sky/catalog/aws_catalog.py:188-201), which is the catalog after
`_fetch_and_apply_az_mapping` (:120-185):

    df = df.merge(az_mappings, on=['AvailabilityZone'], how='inner')
    df = df.drop(columns=['AvailabilityZone']).rename(
        columns={'AvailabilityZoneName': 'AvailabilityZone'})

`mapped_frames` restates those two lines on the synthetic catalog;
`run_scenario` runs optimizer_oracle (or reservation_oracle, for scenarios
with a `reservations` inventory) on the result, so everything downstream --
feasibility, zone order, candidates, DP -- is theirs, on the mapped frame.
"""
import json
from typing import Any, Dict

import pandas as pd

from oracle import optimizer_oracle as oo
from oracle import reservation_oracle


def mapped_frames(catalog_spec: Dict[str, Any],
                  mapping_seed: int) -> Dict[str, pd.DataFrame]:
    from skypilot_b200 import synth  # pylint: disable=import-outside-toplevel
    spec = dict(catalog_spec)
    spec.pop('enabled', None)
    frames = synth.make_catalogs(**spec)
    az_mappings = synth.aws_az_mapping(frames['aws'], mapping_seed)
    df = frames['aws']
    df = df.merge(az_mappings, on=['AvailabilityZone'], how='inner')
    df = df.drop(columns=['AvailabilityZone']).rename(
        columns={'AvailabilityZoneName': 'AvailabilityZone'})
    return dict(frames, aws=df)


def _spec(catalog_spec: Dict[str, Any], mapping_seed: int) -> Dict[str, Any]:
    """optimizer_oracle's catalog key for the mapped catalog, filled once."""
    spec = dict(catalog_spec, az_mapping_seed=mapping_seed)
    key = json.dumps(spec, sort_keys=True)
    if key not in oo._catalog_cache:  # pylint: disable=protected-access
        enabled = catalog_spec.get('enabled') or list(
            catalog_spec.get('clouds') or []) or None
        oo._catalog_cache[key] = oo.Catalog(  # pylint: disable=protected-access
            mapped_frames(catalog_spec, mapping_seed), enabled)
    return spec


def run_scenario(catalog_spec: Dict[str, Any], mapping_seed: int,
                 scenario: Dict[str, Any]) -> Dict[str, Any]:
    spec = _spec(catalog_spec, mapping_seed)
    if 'reservations' in scenario:
        return reservation_oracle.run_scenario(spec, scenario)
    return oo.run_scenario(spec, scenario)
