"""Runs tests/scenarios.py specs through skypilot_b200 (the CUDA path) and
returns records shaped like the reference harness output
(oracle/ref_harness/run_reference.py), so the two can be compared field by
field."""
import contextlib
import json
import math
import os
import re
from typing import Any, Dict, List, Optional

import networkx as nx

import skypilot_b200 as sky
from skypilot_b200 import engine
from skypilot_b200 import optimizer as opt_lib
from skypilot_b200 import synth
from skypilot_b200 import workloads
from tests import scenarios

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
_loaded: Dict[str, Any] = {}
_ANSI = re.compile(r'\x1b\[[0-9;]*m')


def load_golden(name: str) -> Dict[str, Any]:
    with open(os.path.join(GOLDEN_DIR, f'{name}.json'), encoding='utf-8') as f:
        return json.load(f)


def activate_catalog(spec: Dict[str, Any]):
    """Builds (once per spec) and activates the synthetic catalog."""
    key = json.dumps(spec, sort_keys=True)
    store = _loaded.get(key)
    if store is None:
        spec = dict(spec)
        enabled = spec.pop('enabled', None)
        frames = synth.make_catalogs(**spec)
        from skypilot_b200.catalog.store import CatalogStore
        store = CatalogStore.from_frames(frames)
        store.enabled = enabled
        store.set_accelerator_metadata(synth.accelerator_metadata())
        for cloud, frame in synth.images(frames).items():
            store.set_images(cloud, frame)
        _loaded[key] = store
    sky.catalog.set_store(store)
    sky.check.set_enabled_clouds(
        getattr(store, 'enabled', None) or sky.check.ALL_CATALOG_CLOUDS)
    return store


# The chain DP's paths the tests force, by test id, as engine.set_chain_paths
# keywords: the default, the full evaluation on every DAG, the general
# recurrence, both, the chain on the block that places the DAG's last task,
# and that with the full evaluation.
CHAIN_PATHS = {
    None: {},
    '8': {'full': True},
    '16': {'general': True},
    '24': {'full': True, 'general': True},
    '32': {'last_task_block': True},
    '40': {'full': True, 'last_task_block': True},
}


@contextlib.contextmanager
def forced_paths(*stores, mode: str = 'auto', chain: Optional[str] = None):
    """Runs the block with the chain DP on path `chain` (a key of
    CHAIN_PATHS; process-wide) and `stores` in scan mode `mode`, then
    restores the defaults."""
    try:
        engine.set_chain_paths(**CHAIN_PATHS[chain])
        for store in stores:
            store.set_scan_mode(mode)
        yield
    finally:
        for store in stores:
            store.set_scan_mode('auto')
        engine.set_chain_paths()


make_time_estimator = workloads.make_time_estimator
build_dag = workloads.build_dag
blocked_list = workloads.blocked_list
res_record = workloads.res_record


def run_scenario(scenario, with_candidates: bool = True) -> Dict[str, Any]:
    """Plan via Optimizer.optimize (fused device path) and, optionally, the
    ordered candidate tables via _estimate_nodes_cost_or_time."""
    if scenario.get('config') is not None and not scenario.get('_in_config'):
        from skypilot_b200 import skypilot_config  # pylint: disable=import-outside-toplevel
        skypilot_config.set_config(scenario['config'])
        try:
            return run_scenario(dict(scenario, _in_config=True),
                                with_candidates)
        finally:
            skypilot_config.set_config(None)
    minimize_cost = scenario.get('minimize', 'cost') == 'cost'
    target = (sky.OptimizeTarget.COST
              if minimize_cost else sky.OptimizeTarget.TIME)
    record: Dict[str, Any] = {'name': scenario['name']}
    try:
        dag, tasks = build_dag(scenario)
        blocked = blocked_list(scenario)
        record['is_chain'] = bool(dag.is_chain())
        Optimizer = opt_lib.Optimizer
        has_list = any(
            t.get('resources_kind') == 'list' or isinstance(tk.resources, list)
            for t, tk in zip(scenario['tasks'], tasks))
        if with_candidates and not has_list:
            Optimizer._add_dummy_source_sink_nodes(dag)
            try:
                topo = list(nx.topological_sort(dag.get_graph()))
                cost_map, _ = Optimizer._estimate_nodes_cost_or_time(
                    topo, minimize_cost, blocked, quiet=True)
                record['candidates'] = [[[
                    str(r.cloud).lower(), r.instance_type, r.region, r.zone,
                    float(v)
                ] for r, v in cost_map[t].items()] for t in tasks]
            finally:
                Optimizer._remove_dummy_source_sink_nodes(dag)
        Optimizer._add_dummy_source_sink_nodes(dag)
        try:
            graph = dag.get_graph()
            topo = list(nx.topological_sort(graph))
            plan = Optimizer._optimize_dag(dag, minimize_cost, blocked,
                                           quiet=True)
            record['plan'] = [res_record(plan[t]) for t in tasks]
            record['total_cost'] = float(
                Optimizer._compute_total_cost(graph, topo, plan))
            record['total_time'] = float(
                Optimizer._compute_total_time(graph, topo, plan))
            record['objective'] = (record['total_cost'] if minimize_cost else
                                   record['total_time'])
        finally:
            Optimizer._remove_dummy_source_sink_nodes(dag)
        # the public entry point must agree
        for t in tasks:
            t.best_resources = None
        Optimizer.optimize(dag, minimize=target, blocked_resources=blocked,
                           quiet=True)
        assert [res_record(t.best_resources) for t in tasks] == record['plan']
    except sky.exceptions.ResourcesUnavailableError as e:
        record['error'] = {
            'type': 'ResourcesUnavailableError',
            'message': str(e)
        }
    except ValueError as e:
        # an invalid request (e.g. an image tag the cloud does not have):
        # the reference raises while the Resources is constructed
        record['error'] = {'type': 'ValueError', 'message': str(e)}
    return record


def check_chain_suites(mode: str = 'auto', chain: Optional[str] = None):
    """Every scenario of two or more tasks of the multi6k and fuzz6k suites
    against the reference's records, with the kernels forced as
    forced_paths does: [(name, first differences)] and the scan form of each
    scenario's last call."""
    bad, forms = [], []
    for cat in ('multi6k', 'fuzz6k'):
        payload = load_golden(cat)
        records = {r['name']: r for r in payload['records']}
        store = activate_catalog(payload['catalog'])
        with forced_paths(store, mode=mode, chain=chain):
            for sc in scenarios.ALL_SUITES[cat]():
                if len(sc['tasks']) < 2:
                    continue
                d = compare(records[sc['name']],
                            run_scenario(sc, with_candidates=False))
                if d:
                    bad.append((sc['name'], d[:2]))
                forms.append(int(engine.LAST_STATS.scan_form))
    return bad, forms


def close(a: float, b: float, rel: float = 1e-6) -> bool:
    if isinstance(a, str) or isinstance(b, str):
        return str(a) == str(b)
    return math.isclose(a, b, rel_tol=rel, abs_tol=1e-12)


def compare(golden: Dict[str, Any], got: Dict[str, Any],
            unordered_candidates: bool = False,
            check_message: bool = True) -> List[str]:
    """Differences between a reference record and ours (empty = parity).

    Index fields (cloud, instance type, region, zone) must be identical,
    costs within 1e-6 relative (BASELINE.json)."""
    diffs: List[str] = []
    if 'error' in golden or 'error' in got:
        g = golden.get('error', {}).get('type')
        o = got.get('error', {}).get('type')
        if g != o:
            diffs.append(f'error: reference {g}, ours {o}: '
                         f'{got.get("error", {}).get("message", "")[:300]}')
            return diffs
        # same exception class AND the same text (SURVEY.md section 8b): the
        # hints and the fuzzy-candidate list are part of the interface
        gm = _ANSI.sub('', golden['error'].get('message', ''))
        om = _ANSI.sub('', got['error'].get('message', ''))
        if check_message and gm != om:
            diffs.append(f'error message:\n  reference {gm!r}\n  ours      {om!r}')
        return diffs
    if 'candidates' in golden and 'candidates' in got:
        for ti, (gc, oc) in enumerate(
                zip(golden['candidates'], got['candidates'])):
            if unordered_candidates:
                # identity, then value: two requests of a set may expand to the
                # same (cloud, instance type, region, zone) at different
                # prices (GCP: one host VM type under two accelerators)
                key = lambda c: ([str(x) for x in c[:4]], float(c[4]))  # noqa: E731
                gc = sorted(gc, key=key)
                oc = sorted(oc, key=key)
            if len(gc) != len(oc):
                diffs.append(f'task {ti}: {len(gc)} candidates in the '
                             f'reference, {len(oc)} ours')
                continue
            for ci, (g, o) in enumerate(zip(gc, oc)):
                if g[:4] != o[:4]:
                    diffs.append(f'task {ti} cand {ci}: {g[:4]} vs {o[:4]}')
                    break
                if not close(g[4], o[4]):
                    diffs.append(f'task {ti} cand {ci} value: {g[4]} vs '
                                 f'{o[4]}')
                    break
    for ti, (g, o) in enumerate(zip(golden['plan'], got['plan'])):
        if g != o:
            diffs.append(f'plan task {ti}: reference {g}, ours {o}')
    for key in ('objective', 'total_cost', 'total_time'):
        if key in golden and key in got and not close(golden[key], got[key]):
            diffs.append(f'{key}: reference {golden[key]}, ours {got[key]}')
    return diffs
