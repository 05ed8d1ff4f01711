"""Catalog entry points: the active store and the per-cloud dispatcher.

`skypilot_b200.catalog.<function>(..., clouds='aws')` mirrors
sky/catalog/__init__.py:19-53 (`_map_clouds_catalog`: import
`<cloud>_catalog`, call the same-named function). The data behind it is ONE
structure-of-arrays table in GPU memory (`store.CatalogStore`), loaded once
per catalog version with `load_frames` / `load_directory`.
"""
import importlib
import os
from typing import Dict, List, Optional, Sequence, Union

from skypilot_b200.catalog.store import CatalogStore

_store: Optional[CatalogStore] = None
_device: int = 0
DEFAULT_CATALOG_DIR = os.path.expanduser('~/.sky/catalogs/v8')


def set_store(store: Optional[CatalogStore], device: int = 0) -> None:
    global _store, _device
    _store = store
    _device = device


def load_frames(frames: Dict[str, 'object'], device: int = 0,
                order: Optional[Sequence[str]] = None,
                aws_az_mapping: Optional['object'] = None) -> CatalogStore:
    """Ingests `{cloud: vms.csv DataFrame}` and makes it the active catalog.
    `aws_az_mapping`: the account's zone mapping (a DataFrame with columns
    AvailabilityZoneName, AvailabilityZone) applied to the AWS frame."""
    store = CatalogStore.from_frames(frames, order=order,
                                     aws_az_mapping=aws_az_mapping)
    set_store(store, device)
    return store


def load_directory(path: str = DEFAULT_CATALOG_DIR, device: int = 0,
                   clouds: Optional[Sequence[str]] = None,
                   aws_user_hash: Optional[str] = None) -> CatalogStore:
    """Loads `<path>/<cloud>/vms.csv`. AWS zone IDs become the account's
    zone names through `<path>/aws/az_mappings-<aws_user_hash>.csv`, or
    without a hash the newest `aws/az_mappings-*.csv`; with no such file the
    IDs stay (sky/catalog/aws_catalog.py:120-185)."""
    store = CatalogStore.from_directory(path, clouds,
                                        aws_user_hash=aws_user_hash)
    set_store(store, device)
    return store


def get_store(required: bool = True) -> Optional[CatalogStore]:
    global _store
    if _store is None and os.path.isdir(DEFAULT_CATALOG_DIR):
        try:
            load_directory(DEFAULT_CATALOG_DIR)
        except FileNotFoundError:
            pass
    if _store is None and required:
        raise RuntimeError(
            'No catalog loaded: call skypilot_b200.catalog.load_frames() or '
            f'load_directory() (default {DEFAULT_CATALOG_DIR}).')
    return _store


def clear_request_level_cache() -> None:
    """Drops the host-side memos kept on the active store (stated request
    plans, accelerator-name sets) — the counterpart of the reference's
    `annotations.clear_request_level_cache()` (tests/conftest.py:51-52).
    Device-resident catalog columns are untouched. (Resources objects pin
    their plan templates too; callers that want a cold start pop
    `_plan_templates` / `_request_key` from them, as bench.py does.)"""
    if _store is not None:
        _store.__dict__.pop('_plan_cache', None)
        _store.__dict__.pop('_acc_set_cache', None)
        _store.__dict__.pop('_set_id_by_obj', None)
        # invalidates what tasks remember of earlier statements
        _store.__dict__['_memo_generation'] = _store.__dict__.get(
            '_memo_generation', 0) + 1


def get_device() -> int:
    return _device


def view(cloud: str):
    store = get_store()
    # one view object per (store, cloud, device): it only holds references
    views = store.__dict__.setdefault('_views', {})
    key = (cloud, _device)
    v = views.get(key)
    if v is None:
        from skypilot_b200.catalog import common  # pylint: disable=import-outside-toplevel
        if not store.has_cloud(cloud):
            raise ValueError(f'cloud {cloud!r} is not in the loaded catalog '
                             f'{[t.name for t in store.clouds]}')
        v = common.CatalogView(store, cloud.lower(), device=_device)
        views[key] = v
    return v


def module_for(cloud: str):
    return importlib.import_module(
        f'skypilot_b200.catalog.{cloud.lower()}_catalog')


def _map_clouds_catalog(clouds: Union[None, str, List[str]], method: str,
                        *args, **kwargs):
    if clouds is None:
        clouds = [t.name for t in get_store().clouds]
    single = isinstance(clouds, str)
    names = [clouds] if single else list(clouds)
    results = []
    for name in names:
        try:
            module = module_for(name)
        except ModuleNotFoundError:
            raise ValueError(
                f'Cannot find module "{name}_catalog" in the catalog.'
            ) from None
        try:
            fn = getattr(module, method)
        except AttributeError:
            raise AttributeError(f'Module "{name}_catalog" does not '
                                 f'implement the "{method}" method') from None
        results.append(fn(*args, **kwargs))
    return results[0] if single else results


def list_accelerators(gpus_only: bool = True, name_filter: Optional[str] = None,
                      region_filter: Optional[str] = None,
                      quantity_filter: Optional[int] = None, clouds=None,
                      case_sensitive: bool = True, all_regions: bool = False,
                      require_price: bool = True):
    """Accelerators offered by the loaded clouds -> {name: [InstanceTypeInfo]}
    (sky/catalog/__init__.py:56-85). The per-row reduction runs on the device
    (`skyopt_list_offerings`, catalog/listing.py)."""
    results = _map_clouds_catalog(clouds, 'list_accelerators', gpus_only,
                                  name_filter, region_filter, quantity_filter,
                                  case_sensitive, all_regions, require_price)
    if not isinstance(results, list):
        results = [results]
    merged: Dict[str, list] = {}
    for result in results:
        for gpu, items in result.items():
            merged.setdefault(gpu, []).extend(items)
    return merged


def list_accelerator_counts(gpus_only: bool = True,
                            name_filter: Optional[str] = None,
                            region_filter: Optional[str] = None,
                            quantity_filter: Optional[int] = None,
                            clouds=None) -> Dict[str, List[float]]:
    """{accelerator: sorted available counts}
    (sky/catalog/__init__.py:88-119)."""
    results = _map_clouds_catalog(clouds, 'list_accelerators', gpus_only,
                                  name_filter, region_filter, quantity_filter,
                                  all_regions=False, require_price=False)
    if not isinstance(results, list):
        results = [results]
    counts: Dict[str, set] = {}
    for result in results:
        for gpu, items in result.items():
            for item in items:
                counts.setdefault(gpu, set()).add(item.accelerator_count)
    return {gpu: sorted(c) for gpu, c in counts.items()}


def get_arch_from_instance_type(instance_type: str, clouds=None):
    return _map_clouds_catalog(clouds, 'get_arch_from_instance_type',
                               instance_type)


def get_local_disk_from_instance_type(instance_type: str, clouds=None):
    return _map_clouds_catalog(clouds, 'get_local_disk_from_instance_type',
                               instance_type)


def instance_type_exists(instance_type: str, clouds=None) -> bool:
    return _map_clouds_catalog(clouds, 'instance_type_exists', instance_type)


def validate_region_zone(region_name, zone_name, clouds=None):
    return _map_clouds_catalog(clouds, 'validate_region_zone', region_name,
                               zone_name)


def get_hourly_cost(instance_type: str, use_spot: bool, region=None,
                    zone=None, clouds=None) -> float:
    return _map_clouds_catalog(clouds, 'get_hourly_cost', instance_type,
                               use_spot, region, zone)


def get_vcpus_mem_from_instance_type(instance_type: str, clouds=None):
    return _map_clouds_catalog(clouds, 'get_vcpus_mem_from_instance_type',
                               instance_type)


def get_default_instance_type(cpus=None, memory=None, disk_tier=None,
                              local_disk=None, region=None, zone=None,
                              use_spot=False, max_hourly_cost=None,
                              clouds=None):
    return _map_clouds_catalog(clouds, 'get_default_instance_type', cpus,
                               memory, disk_tier, local_disk, region, zone,
                               use_spot, max_hourly_cost)


def get_accelerators_from_instance_type(instance_type: str, clouds=None):
    return _map_clouds_catalog(clouds, 'get_accelerators_from_instance_type',
                               instance_type)


def get_instance_type_for_accelerator(acc_name, acc_count, cpus=None,
                                      memory=None, use_spot=False,
                                      local_disk=None, region=None, zone=None,
                                      max_hourly_cost=None, clouds=None):
    return _map_clouds_catalog(clouds, 'get_instance_type_for_accelerator',
                               acc_name, acc_count, cpus, memory, use_spot,
                               local_disk, region, zone, max_hourly_cost)


def get_costs(resources, seconds):
    """`[r.get_cost(s) for r, s in zip(resources, seconds)]` as a float64
    array, bit for bit, priced in one device call (catalog.pricing)."""
    from skypilot_b200.catalog import pricing  # pylint: disable=import-outside-toplevel
    return pricing.get_costs(resources, seconds)


def get_accelerator_hourly_cost(acc_name, acc_count, use_spot, region=None,
                                zone=None, clouds=None) -> float:
    return _map_clouds_catalog(clouds, 'get_accelerator_hourly_cost', acc_name,
                               acc_count, use_spot, region, zone)


def get_region_zones_for_instance_type(instance_type: str, use_spot: bool,
                                       clouds=None):
    return _map_clouds_catalog(clouds, 'get_region_zones_for_instance_type',
                               instance_type, use_spot)


def get_region_zones_for_accelerators(acc_name, acc_count, use_spot,
                                      clouds=None):
    return _map_clouds_catalog(clouds, 'get_region_zones_for_accelerators',
                               acc_name, acc_count, use_spot)


def check_accelerator_attachable_to_host(instance_type: str, accelerators,
                                         zone: Optional[str] = None,
                                         clouds=None) -> None:
    """GCP only: can the accelerators be attached to the host VM
    (sky/catalog/__init__.py:326-338)."""
    _map_clouds_catalog(clouds, 'check_accelerator_attachable_to_host',
                        instance_type, accelerators, zone)


def get_image_id_from_tag(tag: str, region: Optional[str] = None,
                          clouds=None):
    """sky/catalog/__init__.py:372-376."""
    return _map_clouds_catalog(clouds, 'get_image_id_from_tag', tag, region)


def is_image_tag_valid(tag: str, region: Optional[str], clouds=None) -> bool:
    """sky/catalog/__init__.py:379-383."""
    return _map_clouds_catalog(clouds, 'is_image_tag_valid', tag, region)
