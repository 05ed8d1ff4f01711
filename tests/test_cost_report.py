"""How the batch price path packs its device requests
(skypilot_b200.catalog.pricing.pack), checked against the host statements
of the per-item path without a device: instance ids, price column, region
and zone ids, the GCP accelerator request, host rules, and the items left to
Resources.get_cost."""
import numpy as np
import pytest

import skypilot_b200 as sky
from skypilot_b200 import _native
from skypilot_b200 import engine
from skypilot_b200.catalog import pricing
from tests import cost_report_cases as cases
from tests import scenarios

_CATALOGS = ('three4k', 'vsphere3k', 'gpuclouds')


def _expected(store, spec):
    """(instance request or host value, accelerator request / host value /
    None) as the per-item statements would ask them, or None when the item
    belongs to the per-item path."""
    cloud, it = spec['cloud'], spec['instance_type']
    spot = int(spec['use_spot'])
    region, zone = spec['region'], spec['zone']
    if cloud == 'vsphere':
        inst = ('host', 0.0)
    elif cloud == 'gcp' and it == 'TPU-VM':
        inst = ('host', 0)
    else:
        module = sky.catalog.module_for(cloud)
        if zone is not None and not module._impl.supports_zones:  # pylint: disable=protected-access
            return None
        table = store.cloud(cloud)
        if it not in table.inst_index:
            return None
        rid = engine.region_filter_id(table, region)
        zid = engine.zone_exact_id(table, zone)
        if engine.NO_MATCH_ID in (rid, zid):
            return None
        inst = (_native.PRICE_INSTANCE, table.index, table.inst_index[it],
                spot, rid, zid)
    try:
        accs = cases.launched(spec).accelerators
    except ValueError:  # no such instance type: get_cost raises it
        return None
    if accs is None:
        return inst, None
    if cloud != 'gcp':
        return inst, ('host', 0)
    (name, count), = accs.items()
    table = store.cloud('gcp')
    keys = [k for k, (n, c) in enumerate(store.acc_keys)
            if n.lower() == name.lower() and c == float(count)]
    rid = engine.region_exact_id(table, region)
    zid = engine.zone_exact_id(table, zone)
    if len(keys) != 1 or engine.NO_MATCH_ID in (rid, zid):
        return None
    return inst, (_native.PRICE_ACCELERATOR, table.index, keys[0], spot, rid,
                  zid)


def _request(plan, q, host):
    if q < 0:
        return ('host', host)
    return tuple(int(v) for v in plan.queries[q].tolist())


@pytest.mark.parametrize('cat_name', _CATALOGS)
def test_pack_matches_host_statements(cat_name):
    spec = scenarios.CATALOGS[cat_name]
    store = cases.activate(spec)
    specs = cases.random_specs(cases.catalog_frames(spec), 600, seed=11)
    plan = pricing.pack([cases.launched(s) for s in specs], store)
    assert plan.queries.dtype == _native.PRICE_QUERY_DTYPE
    # one request per distinct question
    assert len({tuple(q.tolist()) for q in plan.queries}) == len(plan.queries)
    n_slow = 0
    for i, s in enumerate(specs):
        want = _expected(store, s)
        if want is None:
            assert plan.slow[i], s
            n_slow += 1
            continue
        assert not plan.slow[i], s
        inst, acc = want
        assert _request(plan, plan.inst_q[i], plan.inst_host[i]) == inst, s
        assert bool(plan.has_acc[i]) == (acc is not None), s
        if acc is not None:
            assert _request(plan, plan.acc_q[i], plan.acc_host[i]) == acc, s
    assert 0 < n_slow < len(specs) // 5


def test_pack_routes_the_rest_to_get_cost():
    store = cases.activate(scenarios.CATALOGS['three4k'])
    spec = {'name': 'x', 'duration': 60, 'num_nodes': 1, 'cloud': 'aws',
            'instance_type': store.cloud('aws').inst_names[0],
            'accelerators': None, 'use_spot': False, 'region': None,
            'zone': None}
    lam = dict(spec, cloud='lambda')  # not in the three4k catalog
    no_cloud = sky.Resources()
    dummy = sky.DummyResources()
    gcp_two = dict(spec, cloud='gcp', instance_type=store.cloud(
        'gcp').inst_names[0], accelerators={'V100': 1, 'T4': 1})
    plan = pricing.pack([cases.launched(spec), cases.launched(lam), no_cloud,
                         dummy, cases.launched(gcp_two)], store)
    assert plan.slow.tolist() == [False, True, True, True, True]
    assert len(plan.queries) == 1


def test_empty_batch_launches_nothing():
    store = cases.activate(scenarios.CATALOGS['three4k'])
    hourly, status = engine.price(
        store, np.zeros(0, dtype=_native.PRICE_QUERY_DTYPE))
    assert hourly.shape == status.shape == (0,)
    assert sky.catalog.get_costs([], []).shape == (0,)


def test_records_without_resources_or_fields_fail_alone(caplog):
    """A history record whose resources could not be restored (None) or that
    lacks a field gets 0.0 and the reference's warning; the others are
    still priced. No record here reaches the device."""
    cases.activate(scenarios.CATALOGS['three4k'])
    dummy = sky.DummyResources()
    records = [
        {'name': 'none', 'duration': 3600, 'num_nodes': 1, 'resources': None},
        {'name': 'free', 'duration': 3600, 'num_nodes': 2,
         'resources': dummy},
        {'name': 'no-duration', 'num_nodes': 1, 'resources': dummy},
        {'name': 'no-nodes', 'duration': 60, 'resources': dummy},
        {'name': 'bad-duration', 'duration': None, 'num_nodes': 1,
         'resources': sky.Resources()},
    ]
    with caplog.at_level('WARNING'):
        reports = sky.cost_report(records)
    assert [r['total_cost'] for r in reports] == [0.0, 0, 0.0, 0.0, 0.0]
    assert [r.getMessage() for r in caplog.records] == [
        "Failed to get total cost for cluster none: 'NoneType' object has "
        "no attribute 'get_cost'",
        "Failed to get total cost for cluster no-duration: 'duration'",
        "Failed to get total cost for cluster no-nodes: 'num_nodes'",
        'Failed to get total cost for cluster bad-duration: unsupported '
        "operand type(s) for /: 'NoneType' and 'int'",
    ]
    assert all(r is not rec for r, rec in zip(reports, records))
    with pytest.raises(AttributeError) as err:
        sky.catalog.get_costs([dummy, None], [60, 60])
    assert str(err.value) == "'NoneType' object has no attribute 'get_cost'"
