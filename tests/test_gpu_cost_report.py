"""Batch prices of launched resources (skypilot_b200.catalog.get_costs,
skypilot_b200.cost_report) on the device: totals and warnings of the
unmodified reference's cost_report step (tests/golden/cost_report.json,
oracle/ref_harness/gen_cost_report.py), bit-identity with the per-item
Resources.get_cost loop, one skyopt_price launch per batch, and the
optimizer's plan total."""
import logging
import math

import networkx as nx
import numpy as np
import pytest

import skypilot_b200 as sky
from skypilot_b200 import _native
from skypilot_b200 import engine
from skypilot_b200 import workloads
from tests import cost_report_cases as cases
from tests import scenario_runner as runner

pytestmark = pytest.mark.gpu

_GOLDEN = runner.load_golden('cost_report')

def _per_item_warning(spec, resources, want: str) -> str:
    """The warning our per-item path gives for a record, exactly, where its
    message differs from the reference's today (the per-item path is kept as
    it is): the catalogs of clouds without spot refuse it before looking for
    a price, the zone message spells the cloud's name differently, and the
    GCP accelerator assertion prints the reference's empty frame."""
    head, text = want.split(': ', 1)
    if text.endswith(' does not support spot.'):
        text = (f'No SpotPrice found for instance type '
                f'{spec["instance_type"]!r}.')
    elif text.endswith(' does not support zones.'):
        text = f'{spec["cloud"].capitalize()} does not support zones.'
    elif text.startswith('Empty DataFrame'):
        (acc, count), = resources.accelerators.items()
        text = f'no {acc}:{count} rows in {spec["region"]} / {spec["zone"]}'
    return f'{head}: {text}'


class _NativeCalls:
    """libskyopt seen through a proxy that counts every entry point called,
    where the call is made."""

    def __init__(self, lib):
        self._lib = lib
        self.calls = {}

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if not name.startswith('skyopt_') or name == 'skyopt_last_error':
            return fn

        def counted(*args):
            self.calls[name] = self.calls.get(name, 0) + 1
            return fn(*args)

        return counted


@pytest.fixture
def native_calls(monkeypatch):
    proxy = _NativeCalls(_native.load())
    monkeypatch.setattr(_native, 'load', lambda: proxy)
    return proxy


def _outcome(fn):
    try:
        return fn(), None
    except Exception as e:  # pylint: disable=broad-except
        return None, (type(e), str(e))


@pytest.mark.parametrize('cat_name', sorted(_GOLDEN['catalogs']))
def test_cost_report_matches_reference(cat_name, caplog):
    part = _GOLDEN['catalogs'][cat_name]
    cases.activate(part['catalog'])
    records = cases.history(part['records'])
    with caplog.at_level(logging.WARNING):
        reports = sky.cost_report(records)
    warnings = [r.getMessage() for r in caplog.records
                if r.levelno == logging.WARNING]
    want_warnings = []
    assert len(reports) == len(records)
    for spec, record, report in zip(part['records'], records, reports):
        assert report is not record and report['resources'] is (
            record['resources'])
        got = report['total_cost']
        if spec.get('pandas_all_na'):
            # the reference's spot -> on-demand fallback, priced by the
            # reference's own functions
            assert got == spec['fallback_total'], spec['name']
            continue
        if spec['failed']:
            want_warnings.append((spec, record['resources'], spec['warning']))
            assert got == 0.0, spec['name']
            continue
        want = spec['total_cost']
        assert got == want or (math.isnan(got) and math.isnan(want)), (
            spec['name'], got, want)
    assert len(warnings) == len(want_warnings)
    differ = [(g, w) for g, (spec, res, w) in zip(warnings, want_warnings)
              if g != w and g != _per_item_warning(spec, res, w)]
    assert not differ


def _random_batch(n=6000, seed=2024):
    spec = workloads.CATALOGS['cfg2']
    frames = cases.catalog_frames(spec)
    runner.activate_catalog(spec)
    specs = cases.random_specs(frames, n, seed)
    return specs, [cases.launched(s) for s in specs]


def test_get_costs_bit_identical_to_get_cost_loop():
    specs, resources = _random_batch()
    seconds = [s['duration'] for s in specs]
    want = [_outcome(lambda r=r, s=s: r.get_cost(s))
            for r, s in zip(resources, seconds)]
    failing = [i for i, (_, err) in enumerate(want) if err is not None]
    ok = [i for i, (_, err) in enumerate(want) if err is None]
    assert len(ok) >= 5000 and failing
    got = sky.catalog.get_costs([resources[i] for i in ok],
                                [seconds[i] for i in ok])
    assert got.dtype == np.float64
    want_ok = np.array([want[i][0] for i in ok], dtype=np.float64)
    assert got.view(np.uint64).tolist() == want_ok.view(np.uint64).tolist()
    # a failing item raises what get_cost raises, whatever is around it
    for i in failing:
        lo, hi = max(i - 3, 0), min(i + 4, len(resources))
        batch = [r for k, r in zip(range(lo, hi), resources[lo:hi])
                 if k == i or want[k][1] is None]
        secs = [s for k, s in zip(range(lo, hi), seconds[lo:hi])
                if k == i or want[k][1] is None]
        _, err = _outcome(lambda b=batch, t=secs: sky.catalog.get_costs(b, t))
        assert err == want[i][1], specs[i]


def test_batch_is_one_price_launch(native_calls, monkeypatch):
    specs, resources = _random_batch(n=2000, seed=7)
    solves = []
    real_solve = engine.solve
    monkeypatch.setattr(engine, 'solve',
                        lambda *a, **k: solves.append(1) or real_solve(*a,
                                                                      **k))
    priced = [s['instance_type'] != 'no-such-type.large' and
              s['region'] != 'nowhere-1' and s['zone'] != 'nowhere-1a' and
              s['accelerators'] != {'V100': 3} for s in specs]
    keep = [i for i, p in enumerate(priced) if p and _outcome(
        lambda i=i: resources[i].get_cost(1.0))[1] is None]
    native_calls.calls.clear()
    solves.clear()
    sky.catalog.get_costs([resources[i] for i in keep],
                          [specs[i]['duration'] for i in keep])
    assert native_calls.calls == {'skyopt_price': 1}
    assert not solves


def test_time_optimize_logs_plan_total_with_one_price_call(
        native_calls, monkeypatch, caplog):
    runner.activate_catalog(workloads.CATALOGS['cfg2'])
    dag, _ = workloads.build_dag(
        workloads.chain('cost_total_chain', [dict(t) for t in
                                             workloads.CFG2_TASKS[:5]]))
    prices = []
    real_price = engine.price
    monkeypatch.setattr(engine, 'price',
                        lambda *a, **k: prices.append(1) or real_price(*a,
                                                                      **k))
    with caplog.at_level(logging.INFO):
        sky.Optimizer.optimize(dag, minimize=sky.OptimizeTarget.TIME,
                               quiet=False)
    assert len(prices) == 1
    assert native_calls.calls.get('skyopt_price') == 1
    # the total as the per-task loop computed it
    graph = dag.get_graph()
    topo = list(nx.topological_sort(graph))
    plan = {t: t.best_resources for t in topo}
    total = 0.
    for node in topo:
        execution = (1 * 3600 if node.time_estimator_func is None else
                     node.estimate_runtime(plan[node]))
        total += plan[node].get_cost(execution) * node.num_nodes
        for pred in graph.predecessors(node):
            total += sky.Optimizer._egress_cost_or_time(  # pylint: disable=protected-access
                True, pred, plan[pred], node, plan[node])
    logged = [r.getMessage() for r in caplog.records
              if 'estimated total cost' in r.getMessage()]
    assert logged and f'estimated total cost: ${total:.1f}' in logged[-1]
    got = sky.Optimizer._compute_total_cost(graph, topo, plan)  # pylint: disable=protected-access
    assert got == total
