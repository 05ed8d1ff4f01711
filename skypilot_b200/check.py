"""Which clouds may be used (stand-in for sky/check.py:406-450).

The reference keeps the credential-checked list of `sky check` in its state
database. Here the list is whatever the host application says it is:

  * `set_enabled_clouds([...])` -- an explicit list of cloud names, or
  * `set_enabled_clouds_provider(fn)` -- a callback returning names or Cloud
    objects; a SkyPilot integration binds it to
    `sky.check.get_cached_enabled_clouds_or_refresh` (INTEGRATION.md), or
  * `set_enabled_clouds(ALL_CATALOG_CLOUDS)` -- every cloud the loaded catalog
    has a `vms.csv` for: an explicit opt-in for tests, benchmarks and
    synthetic catalogs, where there are no credentials to check.

Nothing configured means NO cloud is enabled: `Optimizer.optimize` then raises
`NoCloudAccessError` like the reference does before `sky check` has run, and
never places a task on a cloud the user has no access to.
"""
from typing import Any, Callable, List, Optional, Sequence, Union

from skypilot_b200 import exceptions
from skypilot_b200.placement_context import _active

ALL_CATALOG_CLOUDS = '<all clouds of the loaded catalog>'

_enabled: Union[None, str, List[str]] = None
_provider: Optional[Callable[..., Sequence[Any]]] = None


def set_enabled_clouds(names: Union[None, str, Sequence[str]]) -> None:
    """`names`: cloud names, `ALL_CATALOG_CLOUDS`, or None (= nothing
    configured: fall back to the provider, else no cloud)."""
    global _enabled
    if names is None or names == ALL_CATALOG_CLOUDS:
        _enabled = names
    else:
        _enabled = [n.lower() for n in names]


def set_enabled_clouds_provider(
        provider: Optional[Callable[..., Sequence[Any]]]) -> None:
    """`provider(capability=..., raise_if_no_cloud_access=...)` -> cloud names
    or Cloud objects (anything whose str() is a registered cloud name)."""
    global _provider
    _provider = provider


def get_cached_enabled_clouds_or_refresh(capability=None,
                                         raise_if_no_cloud_access: bool = False):
    from skypilot_b200 import catalog  # pylint: disable=import-outside-toplevel
    from skypilot_b200.utils import registry  # pylint: disable=import-outside-toplevel
    names: List[str] = []
    ctx = _active.get()
    if ctx is not None and ctx.enabled_clouds is not None:
        names = list(ctx.enabled_clouds)
    elif _enabled == ALL_CATALOG_CLOUDS:
        store = catalog.get_store(required=False)
        names = [t.name for t in store.clouds] if store is not None else []
    elif _enabled is not None:
        names = list(_enabled)
    elif _provider is not None:
        try:
            got = _provider(capability=capability,
                            raise_if_no_cloud_access=raise_if_no_cloud_access)
        except TypeError:
            got = _provider()
        names = [str(c).lower() for c in got]
    clouds = []
    for name in names:
        if name in registry.CLOUD_REGISTRY or name in getattr(
                registry.CLOUD_REGISTRY, '_aliases', {}):
            clouds.append(registry.CLOUD_REGISTRY.from_str(name))
    if not clouds and raise_if_no_cloud_access:
        raise exceptions.NoCloudAccessError(
            'Cloud access is not set up. Run `sky check`, or tell '
            'skypilot_b200.check which clouds are enabled '
            '(set_enabled_clouds / set_enabled_clouds_provider).')
    return clouds


def check_capability(*args, **kwargs) -> None:
    del args, kwargs
