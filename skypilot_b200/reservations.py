"""Capacity reservations the placement prices in (sky/optimizer.py:259-357).

The reference asks the clouds' APIs, for every launchable, how many reserved
nodes it may consume (Resources.get_reservations_available_resources,
sky/resources.py:1785-1812), and costs a candidate at
`float(hourly * hours) * max(num_nodes - reserved, 0)`. Here the inventory is
injected, like the enabled clouds (`check.py`):

  * `set_reservations([...])` -- the records themselves, or
  * `set_provider(fn)` -- a callback returning them; a SkyPilot integration
    forwards its own cached listings (`aws_utils.
    list_reservations_for_instance_type`, `gcp_utils.
    list_reservations_for_instance_type_in_zone`; INTEGRATION.md).

A record is a `Reservation` (or a dict with its field names). Which records
count follows the reference:

  * nothing counts unless some cloud's config sets `prioritize_reservations`
    or `specific_reservations` (resources_utils.need_to_query_reservations,
    resources_utils.py:425-451); then nothing is queried or uploaded either;
  * AWS records count only when the AWS config enables reservations
    (aws_utils.use_reservations, aws_utils.py:30-43), GCP records only when
    the GCP config does (gcp_utils.py:131-154); every other cloud has none
    (cloud.py:512-525);
  * a targeted AWS reservation (aws.py:1490-1519) and a GCP reservation with
    `specificReservationRequired` (gcp_utils.py:99-110) are consumable only
    when their name is in `specific_reservations`, resolved per (cloud,
    region) by `skypilot_config.get_effective_region_config`;
  * spot candidates and region-level candidates (zone None) get 0;
  * per (cloud, instance type, zone) the reference keeps one count per
    reservation name (a dict) and sums them. GCP keys on the instance type
    of the launchable, which for an accelerator launchable is its host VM.
"""
import dataclasses
from typing import Any, Callable, Dict, Iterable, List, Optional, Tuple

import numpy as np

from skypilot_b200 import _native
from skypilot_b200 import skypilot_config
from skypilot_b200.placement_context import _active

# clouds whose Cloud.get_reservations_available_resources reads reservations
CLOUDS = ('aws', 'gcp')


@dataclasses.dataclass(frozen=True)
class Reservation:
    cloud: str           # 'aws' or 'gcp'
    instance_type: str   # AWS InstanceType; GCP machineType (host VM)
    zone: str            # AvailabilityZone / GCP zone name
    name: str            # AWS CapacityReservationId; GCP name from selfLink
    available: int       # AvailableInstanceCount; GCP count - inUseCount
    targeted: bool = False  # AWS InstanceMatchCriteria == 'targeted';
                            # GCP specificReservationRequired


_records: Optional[Tuple[Reservation, ...]] = None
_provider: Optional[Callable[[], Iterable[Any]]] = None


def as_record(r: Any) -> Reservation:
    if isinstance(r, Reservation):
        return r
    if isinstance(r, dict):
        d = dict(r)
        if 'specific_reservation_required' in d:
            d['targeted'] = d.pop('specific_reservation_required')
        return Reservation(cloud=str(d['cloud']).lower(),
                           instance_type=str(d['instance_type']),
                           zone=str(d['zone']), name=str(d['name']),
                           available=int(d['available']),
                           targeted=bool(d.get('targeted', False)))
    raise TypeError(f'not a reservation record: {r!r}')


def set_reservations(records: Optional[Iterable[Any]]) -> None:
    """The inventory (None: ask the provider, if any)."""
    global _records
    _records = (None if records is None else tuple(
        as_record(r) for r in records))


def set_provider(provider: Optional[Callable[[], Iterable[Any]]]) -> None:
    """`provider()` -> records; called once per optimisation that needs the
    inventory."""
    global _provider
    _provider = provider


def records() -> Tuple[Reservation, ...]:
    ctx = _active.get()
    if ctx is not None and ctx.reservations is not None:
        return ctx.reservations
    if _records is not None:
        return _records
    if _provider is not None:
        return tuple(as_record(r) for r in _provider())
    return ()


def _config(cloud: str, region: Optional[str], key: str, default: Any) -> Any:
    return skypilot_config.get_effective_region_config(
        cloud=cloud, region=region, keys=(key,), default_value=default)


def cloud_uses_reservations(cloud: str) -> bool:
    """The cloud's own listing is non-empty only under this condition
    (aws_utils.use_reservations; gcp_utils._list_reservations_for_...)."""
    return bool(_config(cloud, None, 'prioritize_reservations', False) or
                _config(cloud, None, 'specific_reservations', None))


def need_to_query() -> bool:
    """resources_utils.need_to_query_reservations (resources_utils.py:
    425-451) over every registered cloud."""
    from skypilot_b200.utils import registry  # pylint: disable=import-outside-toplevel
    for cloud in registry.CLOUD_REGISTRY.keys():
        if (_config(cloud, None, 'specific_reservations', None) is not None or
                _config(cloud, None, 'prioritize_reservations', False)):
            return True
    return False


def specific_reservations(cloud: str, region: Optional[str]) -> set:
    """Resources.get_reservations_available_resources' name set."""
    return set(_config(cloud, region, 'specific_reservations', set()) or ())


def available(cloud: str, instance_type: Optional[str], region: Optional[str],
              zone: Optional[str], use_spot: bool,
              inventory: Optional[Iterable[Reservation]] = None) -> int:
    """sum(Resources.get_reservations_available_resources().values()) of one
    launchable, as the reference's optimizer sees it."""
    cloud = cloud.lower()
    if (use_spot or zone is None or cloud not in CLOUDS or
            not need_to_query() or not cloud_uses_reservations(cloud)):
        return 0
    names = specific_reservations(cloud, region)
    by_name: Dict[str, int] = {}
    for r in (records() if inventory is None else inventory):
        if (r.cloud == cloud and r.instance_type == instance_type and
                r.zone == zone and (not r.targeted or r.name in names)):
            by_name[r.name] = r.available
    return sum(by_name.values())


def snapshot() -> Optional[Tuple[Any, ...]]:
    """What a solve depends on: None when nothing is queried, else the
    inventory and the configuration's key (skypilot_config.key)."""
    if not need_to_query():
        return None
    return (records(), skypilot_config.key())


def device_table(store, snap: Optional[Tuple[Any, ...]]) -> np.ndarray:
    """The consumable counts of `snap` as SkyoptReservation rows, one per
    (cloud, instance type, zone) of the catalog, sorted by those ids.
    Records naming an instance type or zone the catalog lacks match no
    candidate and are left out."""
    rows: Dict[Tuple[int, int, int], Dict[str, int]] = {}
    if snap is not None:
        for r in snap[0]:
            if r.cloud not in CLOUDS or not store.has_cloud(r.cloud):
                continue
            if not cloud_uses_reservations(r.cloud):
                continue
            table = store.cloud(r.cloud)
            inst = table.inst_index.get(r.instance_type)
            zone = table.zone_exact.get(r.zone) if table.has_zone_column else None
            if inst is None or zone is None:
                continue
            region = table.region_names[table.zone_region[zone]]
            if r.targeted and r.name not in specific_reservations(r.cloud,
                                                                  region):
                continue
            rows.setdefault((table.index, inst, zone), {})[r.name] = r.available
    keys = sorted(rows)
    out = np.zeros(len(keys), dtype=_native.RESERVATION_DTYPE)
    for i, k in enumerate(keys):
        out[i] = k + (sum(rows[k].values()),)
    return out


def clouds_in(table: np.ndarray) -> List[int]:
    return sorted(set(int(c) for c in table['cloud']))
