"""The few look-ups of sky/skypilot_config.py the placement path makes.

Only one key matters to the optimizer: a per-region `ssh_proxy_command`
restricts a cloud's usable regions to the dict's keys
(Resources.get_valid_regions_for_launchable, sky/resources.py:1210-1246):

    aws:
      ssh_proxy_command:
        us-east-1: ssh -W %h:%p jump-east
        eu-west-1: ssh -W %h:%p jump-eu

The configuration is a nested dict: `load()` reads `~/.sky/config.yaml` (or
$SKYPILOT_CONFIG) like the reference, `set_config` / `set_nested` install one
directly (a SkyPilot integration forwards its own `skypilot_config` dict).
Every change bumps a generation counter that is part of the statement memos'
keys. An active placement context (placement_context.py) with a config of
its own replaces the process-wide one; the memos then key on its content."""
import copy
import os
from typing import Any, Dict, Hashable, Optional, Tuple

from skypilot_b200.placement_context import _active

_config: Dict[str, Any] = {}
_generation = 0
ENV_VAR = 'SKYPILOT_CONFIG'
DEFAULT_PATH = '~/.sky/config.yaml'


def generation() -> int:
    return _generation


def key() -> Hashable:
    """What statements depend on: the content of the active context's
    config, else the process-wide generation."""
    ctx = _active.get()
    if ctx is not None and ctx.config is not None:
        return ctx.config_key
    return _generation


def _current() -> Dict[str, Any]:
    ctx = _active.get()
    if ctx is not None and ctx.config is not None:
        return ctx.config
    return _config


def _changed() -> None:
    global _generation
    _generation += 1


def has_config() -> bool:
    return bool(_current())


def set_config(config: Optional[Dict[str, Any]]) -> None:
    global _config
    _config = copy.deepcopy(config) if config else {}
    _changed()


def load(path: Optional[str] = None) -> Dict[str, Any]:
    """Reads a SkyPilot config file (YAML); a missing file is an empty
    config."""
    import yaml  # pylint: disable=import-outside-toplevel
    path = os.path.expanduser(path or os.environ.get(ENV_VAR) or DEFAULT_PATH)
    data: Dict[str, Any] = {}
    if os.path.exists(path):
        with open(path, encoding='utf-8') as f:
            data = yaml.safe_load(f) or {}
    set_config(data)
    return data


def get_nested(keys: Tuple[str, ...], default_value: Any = None) -> Any:
    cur: Any = _current()
    for k in keys:
        if not isinstance(cur, dict) or k not in cur:
            return default_value
        cur = cur[k]
    return cur


def set_nested(keys: Tuple[str, ...], value: Any) -> None:
    cur = _config
    for k in keys[:-1]:
        cur = cur.setdefault(k, {})
    cur[keys[-1]] = copy.deepcopy(value)
    _changed()


def get_effective_region_config(cloud: str, region: Optional[str],
                                keys: Tuple[str, ...],
                                default_value: Any = None) -> Any:
    """`<cloud>.<keys...>` (sky/skypilot_config.py get_effective_region_config,
    sky/utils/config_utils.py:281-330). A per-region override
    `<cloud>.region_configs.<region>.<keys...>` replaces the cloud-level
    value for the clouds the reference reads it for (Nebius, OCI); for every
    other catalog cloud the cloud-level value applies in every region (the
    Kubernetes / SSH context layer has no catalog and is out of scope)."""
    keys = tuple(keys)
    if region is not None and cloud in _REGION_CONFIG_CLOUDS:
        override = get_nested((cloud, 'region_configs', region) + keys, None)
        if override is not None:
            return override
    return get_nested((cloud,) + keys, default_value)


_REGION_CONFIG_CLOUDS = ('nebius', 'oci')


def allowed_regions_by_ssh_proxy(cloud: str) -> Optional[set]:
    """Region names a per-region ssh_proxy_command allows, or None (no
    restriction: unset, or one command for every region)."""
    cfg = get_effective_region_config(cloud=cloud, region=None,
                                      keys=('ssh_proxy_command',),
                                      default_value=None)
    if cfg is None or isinstance(cfg, str):
        return None
    return set(cfg.keys())
