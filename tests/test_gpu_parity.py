"""CUDA path vs the unmodified reference (committed golden fixtures).

For every scenario of tests/scenarios.py the fused device path must return
the reference's plan (cloud, instance type, region, zone: identical), the
ordered candidate tables of every task (identical order and identity, values
within 1e-6 relative) and the objective / total cost / total time.
"""
import json
import os

import pytest

import skypilot_b200 as sky
from tests import scenario_runner as runner
from tests import scenarios

pytestmark = pytest.mark.gpu


def _cases():
    out = []
    for catalog in scenarios.SUITES:
        # a missing fixture is a failure (load_golden raises), never a skip
        for sc in scenarios.SUITES[catalog]():
            out.append(pytest.param(catalog, sc, id=f'{catalog}:{sc["name"]}'))
    return out


_golden_cache = {}


def _golden(catalog):
    if catalog not in _golden_cache:
        payload = runner.load_golden(catalog)
        _golden_cache[catalog] = (payload['catalog'], {
            r['name']: r for r in payload['records']
        })
    return _golden_cache[catalog]


@pytest.mark.parametrize('catalog,scenario', _cases())
def test_scenario_matches_reference(catalog, scenario):
    spec, records = _golden(catalog)
    assert spec == scenarios.CATALOGS[catalog], (
        'fixture was generated for a different catalog spec; rerun '
        'oracle/ref_harness/gen_golden.py')
    golden = records[scenario['name']]
    runner.activate_catalog(spec)
    got = runner.run_scenario(scenario)
    unordered = any(
        t.get('resources_kind') == 'set' for t in scenario['tasks'])
    diffs = runner.compare(golden, got, unordered_candidates=unordered)
    if diffs:
        out = os.path.join(os.path.dirname(runner.GOLDEN_DIR), '..',
                           'gpurun_out')
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, 'parity_failures.jsonl'), 'a',
                  encoding='utf-8') as f:
            f.write(json.dumps({'catalog': catalog, 'name': scenario['name'],
                                'diffs': diffs, 'got': got}) + '\n')
    assert not diffs, '\n'.join(diffs)


@pytest.mark.parametrize('mode', ['tile', 'queue',
                                  'queue32', 'fast-noprune',
                                  'fast-split', 'fast-split-noprune'])
@pytest.mark.parametrize('catalog', ['multi50k', 'aws50k'])
def test_scan_kernel_variants_agree_with_reference(catalog, mode):
    """All scan kernels (one tile per block / the queue form with few and
    with 32 tiles per block / the class-table scan with and without pruning)
    must give the reference's answers."""
    spec, records = _golden(catalog)
    store = runner.activate_catalog(spec)
    store.set_scan_mode(mode)
    try:
        failures = []
        for sc in scenarios.SUITES[catalog]():
            got = runner.run_scenario(sc)
            unordered = any(
                t.get('resources_kind') == 'set' for t in sc['tasks'])
            diffs = runner.compare(records[sc['name']], got, unordered)
            if diffs:
                failures.append((sc['name'], diffs[:3]))
        assert not failures, failures
    finally:
        store.set_scan_mode('auto')


def test_retired_scan_modes_are_rejected():
    """Modes 2 and 3 (the retired TMA streaming scan) and 6 (the class-table
    scan as `auto` runs it) fail with SKYOPT_EINVAL and leave the catalog's
    mode alone; the Python API no longer names them. The SKYOPT_SPLIT
    environment variable no longer selects separate launches."""
    import subprocess
    import sys
    from skypilot_b200 import _native
    spec, records = _golden('multi6k')
    store = runner.activate_catalog(spec)
    lib = _native.load()
    for code in (2, 3, 6):
        assert lib.skyopt_catalog_set_scan_mode(store.handle(0), code) == -1
        assert b'removed' in lib.skyopt_last_error()
    for name in ('stream', 'stream3', 'fast'):
        with pytest.raises(KeyError):
            store.set_scan_mode(name)
    sc = next(s for s in scenarios.SUITES['multi6k']()
              if s['name'] == 'chain3_mixed')
    assert not runner.compare(records[sc['name']], runner.run_scenario(sc))
    code = (
        'import sys; sys.path.insert(0, ".")\n'
        'from tests import scenario_runner as runner, scenarios\n'
        'from skypilot_b200 import engine\n'
        'runner.activate_catalog(scenarios.CATALOGS["multi6k"])\n'
        'sc = next(s for s in scenarios.SUITES["multi6k"]()\n'
        '          if s["name"] == "chain3_mixed")\n'
        'runner.run_scenario(sc, with_candidates=False)\n'
        'print("form", int(engine.LAST_STATS.scan_form))\n')
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    proc = subprocess.run([sys.executable, '-c', code], cwd=root,
                          env=dict(os.environ, SKYOPT_SPLIT='1'),
                          capture_output=True, text=True, timeout=600,
                          check=False)
    assert proc.returncode == 0, proc.stdout[-2000:] + proc.stderr[-2000:]
    assert 'form 4' in proc.stdout.splitlines()[-1], proc.stdout[-2000:]


def test_auto_mode_takes_the_class_table_scan():
    """`auto` must run the fused step_kernel (SkyoptStats.scan_form 4: class-
    table scan, placement and chain DP in one cooperative launch), not
    silently fall back to the round-1 kernels."""
    from skypilot_b200 import engine
    spec, records = _golden('multi6k')
    runner.activate_catalog(spec)
    sc = next(s for s in scenarios.SUITES['multi6k']()
              if s['name'] == 'chain3_mixed')
    got = runner.run_scenario(sc, with_candidates=False)
    assert not runner.compare(records[sc['name']], got)
    assert engine.LAST_STATS is not None
    assert int(engine.LAST_STATS.scan_form) == 4
    assert int(engine.LAST_STATS.total_launches) == 1


@pytest.mark.parametrize('path,mode', [
    pytest.param(path, mode, id=path if mode == 'auto' else f'{mode}-{path}')
    for mode in ('auto', 'fast-split', 'tile') for path in ('8', '16', '24')
])
def test_chain_dp_code_paths_agree(path, mode):
    """The chain DP works on per-cloud minima and only reads the candidate
    tables after a rounding hazard; with at most four clouds and
    non-negative values it runs a shorter recurrence (skyopt_step.cuh).
    8 forces the full evaluation on every DAG, 16 the general recurrence, 24
    both: same plans, same objectives, in the fused step (`auto`) and in
    solve_kernel after separate launches (`fast-split`, `tile`)."""
    bad, forms = runner.check_chain_suites(mode, path)
    # any mode but auto: solve_kernel, not the fused step (form 4)
    assert set(forms) <= ({0, 1, 2, 3, 4} if mode == 'auto' else
                          {0, 1, 2, 3}), forms
    assert not bad, bad


def test_fresh_request_with_equal_content_hits_the_statement_memo():
    """A new DAG (new Task / Resources objects) whose requests have the same
    content as an earlier one replays the stated plans kept on the catalog
    store -- the memo is keyed by request content, not by object identity --
    and still gives the reference's record."""
    spec, records = _golden('multi6k')
    store = runner.activate_catalog(spec)
    sky.catalog.clear_request_level_cache()
    sc = next(s for s in scenarios.SUITES['multi6k']()
              if s['name'] == 'chain3_mixed')
    first = runner.run_scenario(sc, with_candidates=False)
    assert not runner.compare(records[sc['name']], first)
    cache = store.__dict__['_plan_cache']
    stated = len(cache)
    assert stated > 0
    # what the rule code costs is what the memo saves: it must not run again
    from skypilot_b200.clouds import cloud as cloud_lib
    calls = []
    original = cloud_lib.Cloud._feature_hint  # pylint: disable=protected-access

    def counting(self, resources, num_nodes):
        calls.append(type(self).__name__)
        return original(self, resources, num_nodes)

    cloud_lib.Cloud._feature_hint = counting  # pylint: disable=protected-access
    try:
        again = runner.run_scenario(sc, with_candidates=False)  # fresh objects
    finally:
        cloud_lib.Cloud._feature_hint = original  # pylint: disable=protected-access
    assert not calls, calls
    assert len(store.__dict__['_plan_cache']) == stated
    assert not runner.compare(records[sc['name']], again)
    assert again['plan'] == first['plan']
