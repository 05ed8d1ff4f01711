"""What a plan depends on besides the DAG: the placement context.

A controller or API server that plans launches for many users has no single
set of enabled clouds, SkyPilot config, reservation inventory or objective:
each workspace enables its own clouds, each request carries its user's
config. `PlacementContext` names those four for one DAG of
`Optimizer.optimize_batch(..., contexts=[...])`; a field left `None` is the
process-wide value (`check.set_enabled_clouds`, `skypilot_config.set_config`,
`reservations.set_reservations`, the call's `minimize`), read as before.

While a context is active (`active(ctx)`), `check`, `skypilot_config` and
`reservations` answer from it. The active context lives in a
`contextvars.ContextVar`: it is private to the thread (and asyncio task)
that set it, and a thread started while it is set does not inherit it.
"""
import contextlib
import contextvars
import copy
import json
from typing import Any, Iterator, Optional, Sequence, Tuple


class PlacementContext:
    """The enabled clouds, SkyPilot config, reservation inventory and
    objective of one DAG of a batch; `None` = the process-wide value.

    `enabled_clouds`: cloud names or `Cloud` objects (an empty list enables
    nothing: that DAG fails with NoCloudAccessError). `config`: a SkyPilot
    config dict (copied). `reservations`: records as
    `reservations.set_reservations` takes them. `minimize`: an
    `OptimizeTarget`."""

    __slots__ = ('enabled_clouds', 'config', 'reservations', 'minimize',
                 'config_key')

    def __init__(self,
                 enabled_clouds: Optional[Sequence[Any]] = None,
                 config: Optional[dict] = None,
                 reservations: Optional[Sequence[Any]] = None,
                 minimize: Any = None):
        from skypilot_b200 import reservations as resv_lib  # pylint: disable=import-outside-toplevel
        self.enabled_clouds: Optional[Tuple[str, ...]] = (
            None if enabled_clouds is None else tuple(
                str(c).lower() for c in enabled_clouds))
        self.config: Optional[dict] = (None if config is None else
                                       copy.deepcopy(dict(config)))
        # what the statement memos key on: the config's content, so that
        # contexts with equal configs share statements
        self.config_key: Optional[str] = (None if config is None else
                                          config_content_key(self.config))
        self.reservations = (None if reservations is None else tuple(
            resv_lib.as_record(r) for r in reservations))
        self.minimize = minimize

    def __repr__(self) -> str:
        return (f'PlacementContext(enabled_clouds={self.enabled_clouds!r}, '
                f'config={self.config!r}, reservations={self.reservations!r},'
                f' minimize={self.minimize!r})')


def config_content_key(config: dict) -> str:
    """A canonical text of a config dict: equal for equal contents."""

    def default(o):
        if isinstance(o, (set, frozenset)):
            return sorted(o, key=repr)
        return repr(o)

    return 'config:' + json.dumps(config, sort_keys=True, default=default)


_active: contextvars.ContextVar[Optional[PlacementContext]] = (
    contextvars.ContextVar('skypilot_b200_placement_context', default=None))


def current() -> Optional[PlacementContext]:
    """The active context, or None (every value is process-wide)."""
    return _active.get()


@contextlib.contextmanager
def active(ctx: Optional[PlacementContext]) -> Iterator[None]:
    """Makes `ctx` the active context of this thread for the block (None:
    the process-wide values)."""
    token = _active.set(ctx)
    try:
        yield
    finally:
        _active.reset(token)
