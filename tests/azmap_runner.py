"""Runs the zone-mapping scenarios (tests/azmap_scenarios.py) through
skypilot_b200 on the mapped catalog and compares them with the reference's
records (tests/golden/azmap.json, tests/golden/azmap_reservations.json):
plans, ordered candidate tables and DP objectives bit-equal, error texts
character-equal."""
from typing import Any, Dict, List

import skypilot_b200 as sky
from skypilot_b200 import synth
from skypilot_b200.catalog.store import CatalogStore
from tests import azmap_scenarios
from tests import reservation_runner
from tests import scenario_runner as runner

_stores: Dict[str, CatalogStore] = {}


def golden(name: str = 'azmap') -> Dict[str, Any]:
    payload = runner.load_golden(name)
    assert payload['catalog'] == azmap_scenarios.CATALOG
    assert payload['az_mapping_seed'] == azmap_scenarios.AZ_MAPPING_SEED
    return payload


def records(name: str = 'azmap') -> Dict[str, Dict[str, Any]]:
    return {r['name']: r for r in golden(name)['records']}


def build_store() -> CatalogStore:
    """The azmap catalog ingested with the account's mapping."""
    frames, mapping = azmap_scenarios.frames_and_mapping()
    store = CatalogStore.from_frames(frames, aws_az_mapping=mapping)
    store.set_accelerator_metadata(synth.accelerator_metadata())
    for cloud, frame in synth.images(frames).items():
        store.set_images(cloud, frame)
    return store


def activate() -> CatalogStore:
    store = _stores.get('azmap')
    if store is None:
        store = _stores['azmap'] = build_store()
    sky.catalog.set_store(store)
    sky.check.set_enabled_clouds(azmap_scenarios.CATALOG['clouds'])
    return store


def optimizer_scenarios() -> List[Dict[str, Any]]:
    return (azmap_scenarios.azmap_scenarios() +
            azmap_scenarios.reservation_scenarios())


def check_all() -> List[Any]:
    """Every optimizer record of both fixtures; the differences found."""
    want = dict(records('azmap'), **records('azmap_reservations'))
    activate()
    bad = []
    for sc in optimizer_scenarios():
        d = reservation_runner.diffs(want[sc['name']],
                                     reservation_runner.run(sc))
        if d:
            bad.append((sc['name'], d[:3]))
    return bad
