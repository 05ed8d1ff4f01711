"""Prices of many launched resources in one device call.

`get_costs(resources, seconds)` is `[r.get_cost(s) for r, s in ...]` with the
catalog look-ups of every item batched into one `skyopt_price` launch; the
arithmetic stays get_cost's (sky/resources.py:1685-1698): instance price,
plus the accelerator price where the cloud adds one, times the hours.
`cost_report(records)` is the per-record step of sky.core.cost_report
(sky/core.py:446-468) on top of it.

What the device answers is decided per item by `pack`: the catalog rows of an
instance type (get_hourly_cost_impl, common.py:360-400) and of a GCP
accelerator (get_accelerator_hourly_cost, gcp_catalog.py:424-442). Host rules
stay host rules -- clouds that override the instance price (vSphere's zero
price), GCP's `TPU-VM` host, the zero accelerator price of every other cloud.
Every other item, and every item whose request the device could not price,
goes through the per-item `Resources.get_cost`, which raises what it raises
today; only those items pay for it.
"""
import logging
from typing import Any, Dict, List, NamedTuple, Optional, Sequence, Tuple

import numpy as np

from skypilot_b200 import _native
from skypilot_b200 import engine
from skypilot_b200.clouds import cloud as cloud_lib

logger = logging.getLogger(__name__)

# a request answered on the host: (_HOST, value of that price part)
_HOST = 'host'
_UNSEEN = object()


class PricePlan(NamedTuple):
    """What `pack` made of a batch. Per item: the request index of its
    instance price (-1: `inst_host` holds it), of its accelerator price (-1:
    `acc_host` holds it, or `has_acc` is False) and whether it takes the
    per-item path (`slow`)."""
    queries: np.ndarray  # PRICE_QUERY_DTYPE, one per distinct request
    inst_q: np.ndarray
    inst_host: np.ndarray
    has_acc: np.ndarray
    acc_q: np.ndarray
    acc_host: np.ndarray
    slow: np.ndarray


def _catalog_impl(cloud):
    """(the CloudCatalog behind a cloud's catalog module or None, the
    module)."""
    module = cloud._catalog_module()  # pylint: disable=protected-access
    impl = getattr(module, '_impl', None)
    if impl is None:
        return None, module
    return impl, module


def _table(store, impl):
    if store is None or impl is None or not store.has_cloud(impl.cloud):
        return None
    return store.cloud(impl.cloud)


def _instance_request(store, r) -> Optional[Any]:
    """(kind, cloud, id, col, region, zone), a host value, or None for the
    per-item path: the statements of Cloud.instance_type_to_hourly_cost ->
    CloudCatalog.get_hourly_cost -> common.get_hourly_cost_impl."""
    cloud = r.cloud
    instance_type = r.instance_type
    if type(cloud).instance_type_to_hourly_cost is not (
            cloud_lib.Cloud.instance_type_to_hourly_cost):
        # a host rule (vSphere: every instance costs 0.0)
        return (_HOST, cloud.instance_type_to_hourly_cost(
            instance_type, r.use_spot, r.region, r.zone))
    impl, module = _catalog_impl(cloud)
    if impl is None:
        return None
    if module.__name__.endswith('.gcp_catalog') and instance_type == 'TPU-VM':
        # the TPU VM host is not billed separately
        return (_HOST, module.get_hourly_cost(instance_type, r.use_spot,
                                              r.region, r.zone))
    if module.get_hourly_cost != impl.get_hourly_cost and not (
            module.__name__.endswith('.gcp_catalog')):
        return None
    if r.zone is not None and not impl.supports_zones:
        return None
    table = _table(store, impl)
    if table is None:
        return None
    inst = table.inst_index.get(instance_type)
    if inst is None:
        return None
    region = engine.region_filter_id(table, r.region)
    zone = engine.zone_exact_id(table, r.zone)
    if engine.NO_MATCH_ID in (region, zone):
        return None
    return (_native.PRICE_INSTANCE, table.index, inst, int(bool(r.use_spot)),
            region, zone)


def _accelerator_request(store, r, accelerators) -> Optional[Any]:
    """As _instance_request, for Cloud.accelerators_to_hourly_cost: zero on
    every cloud but GCP, whose accelerator-only rows the device prices."""
    from skypilot_b200.clouds import gcp  # pylint: disable=import-outside-toplevel
    cloud = r.cloud
    method = type(cloud).accelerators_to_hourly_cost
    if method is not gcp.GCP.accelerators_to_hourly_cost:
        return (_HOST, cloud.accelerators_to_hourly_cost(
            accelerators, r.use_spot, r.region, r.zone))
    if len(accelerators) != 1:
        return None
    impl, module = _catalog_impl(cloud)
    table = _table(store, impl)
    if table is None or not module.__name__.endswith('.gcp_catalog'):
        return None
    name, count = list(accelerators.items())[0]
    _, _, strict = engine.accelerator_sets(store, name, count)
    keys = np.flatnonzero(np.unpackbits(strict.view(np.uint8),
                                        bitorder='little'))
    if len(keys) != 1:
        # no row at all (a NaN price or the reference's assertion) or
        # several keys: the per-item path
        return None
    region = engine.region_exact_id(table, r.region)
    zone = engine.zone_exact_id(table, r.zone)
    if engine.NO_MATCH_ID in (region, zone):
        return None
    return (_native.PRICE_ACCELERATOR, table.index, int(keys[0]),
            int(bool(r.use_spot)), region, zone)


def _item_key(r) -> Optional[Tuple]:
    """What an item's requests depend on, or None when it is not
    Resources.get_cost that prices it (a subclass with its own, or no
    Resources at all, such as the None of a history record whose resources
    could not be restored) or its fields do not make a key: such items take
    the per-item path, which raises what the per-item loop raises."""
    from skypilot_b200 import resources as resources_lib  # pylint: disable=import-outside-toplevel
    if not isinstance(r, resources_lib.Resources) or (
            type(r).get_cost is not resources_lib.Resources.get_cost):
        return None
    try:
        acc = r._accelerators  # pylint: disable=protected-access
        key = (type(r.cloud), r.instance_type, bool(r.use_spot), r.region,
               r.zone, None if acc is None else tuple(acc.items()))
        hash(key)
    except Exception:  # pylint: disable=broad-except
        return None
    return key


def pack(resources: Sequence[Any], store) -> PricePlan:
    """The device requests of a batch and how each item uses them."""
    n = len(resources)
    inst_q = np.full(n, -1, dtype=np.int64)
    acc_q = np.full(n, -1, dtype=np.int64)
    inst_host = np.zeros(n, dtype=np.float64)
    acc_host = np.zeros(n, dtype=np.float64)
    has_acc = np.zeros(n, dtype=bool)
    slow = np.zeros(n, dtype=bool)
    requests: Dict[Tuple, int] = {}
    # items that differ only in duration share their requests
    plans: Dict[Tuple, Optional[Tuple]] = {}

    def index(req) -> int:
        if req[0] == _HOST:
            return -1
        return requests.setdefault(req, len(requests))

    for i, r in enumerate(resources):
        key = _item_key(r)
        plan = plans.get(key, _UNSEEN) if key is not None else None
        if plan is _UNSEEN:
            plan = None
            if r.cloud is not None and r.instance_type is not None:
                try:
                    inst = _instance_request(store, r)
                    acc = None
                    accelerators = r.accelerators if inst is not None else None
                    if accelerators is not None:
                        acc = _accelerator_request(store, r, accelerators)
                    if inst is not None and (accelerators is None or
                                             acc is not None):
                        plan = (inst, accelerators is not None, acc)
                except Exception:  # pylint: disable=broad-except
                    # get_cost raises it again, on the per-item path
                    plan = None
            plans[key] = plan
        if plan is None:
            slow[i] = True
            continue
        inst, with_acc, acc = plan
        inst_q[i] = index(inst)
        if inst_q[i] < 0:
            inst_host[i] = inst[1]
        has_acc[i] = with_acc
        if with_acc:
            acc_q[i] = index(acc)
            if acc_q[i] < 0:
                acc_host[i] = acc[1]
    queries = np.zeros(len(requests), dtype=_native.PRICE_QUERY_DTYPE)
    if requests:
        queries[:] = list(requests.keys())
    return PricePlan(queries, inst_q, inst_host, has_acc, acc_q, acc_host,
                     slow)


def _costs(resources: Sequence[Any], seconds: Sequence[float],
           stop_at_error: bool) -> Tuple[np.ndarray, Dict[int, Exception]]:
    from skypilot_b200 import catalog  # pylint: disable=import-outside-toplevel
    n = len(resources)
    if len(seconds) != n:
        raise ValueError(f'{n} resources but {len(seconds)} durations')
    store = catalog.get_store(required=False)
    plan = pack(resources, store)
    hourly_q, status = engine.price(store, plan.queries, catalog.get_device())
    slow = plan.slow.copy()
    inst = plan.inst_host.copy()
    dev = plan.inst_q >= 0
    inst[dev] = hourly_q[plan.inst_q[dev]]
    slow[dev] |= status[plan.inst_q[dev]] != _native.PRICE_OK
    acc = plan.acc_host.copy()
    dev = plan.acc_q >= 0
    acc[dev] = hourly_q[plan.acc_q[dev]]
    slow[dev] |= status[plan.acc_q[dev]] != _native.PRICE_OK
    # hourly_cost += accelerators' price only where get_cost adds it
    hourly = np.where(plan.has_acc, inst + acc, inst)
    hours = np.zeros(n, dtype=np.float64)
    for i, s in enumerate(seconds):
        try:
            hours[i] = s / 3600
        except Exception:  # pylint: disable=broad-except
            slow[i] = True  # get_cost raises it again
    out = hourly * hours
    errors: Dict[int, Exception] = {}
    for i in np.flatnonzero(slow):
        try:
            out[i] = resources[i].get_cost(seconds[i])
        except Exception as e:  # pylint: disable=broad-except
            if stop_at_error:
                raise
            errors[int(i)] = e
            out[i] = 0.0
    return out, errors


def get_costs(resources: Sequence[Any],
              seconds: Sequence[float]) -> np.ndarray:
    """`[r.get_cost(s) for r, s in zip(resources, seconds)]` as a float64
    array, bit for bit, with one `skyopt_price` launch for the whole batch.
    Raises what the first failing `get_cost` raises."""
    out, _ = _costs(resources, seconds, stop_at_error=True)
    return out


def cost_report(records: Sequence[Dict[str, Any]]) -> List[Dict[str, Any]]:
    """The per-record step of sky.core.cost_report (sky/core.py:446-468):
    copies of the records (`name`, `duration`, `num_nodes`, `resources`, as
    global_user_state.get_clusters_from_history yields them) with
    `total_cost = resources.get_cost(duration) * num_nodes`; a record whose
    cost cannot be computed gets 0.0 and a warning."""
    reports = [record.copy() for record in records]
    errors: Dict[int, Exception] = {}
    batch: List[int] = []
    fields = []
    for i, report in enumerate(reports):
        try:
            # read in the reference's order (sky/core.py:452-454)
            fields.append((report['duration'], report['num_nodes'],
                           report['resources']))
            batch.append(i)
        except Exception as e:  # pylint: disable=broad-except
            errors[i] = e
    costs, batch_errors = _costs([fields[k][2] for k in range(len(batch))],
                                 [fields[k][0] for k in range(len(batch))],
                                 stop_at_error=False)
    for k, i in enumerate(batch):
        e = batch_errors.get(k)
        if e is None:
            try:
                reports[i]['total_cost'] = float(costs[k]) * fields[k][1]
            except Exception as err:  # pylint: disable=broad-except
                e = err
        if e is not None:
            errors[i] = e
    for i, report in enumerate(reports):
        e = errors.get(i)
        if e is not None:
            # Ok to skip the total cost as this is just for display purposes.
            logger.warning(f'Failed to get total cost for cluster '
                           f'{report["name"]}: {str(e)}')
            report['total_cost'] = 0.0
    return reports
