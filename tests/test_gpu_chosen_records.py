"""A chain DP without a hazard writes each task's chosen candidate record
from the record its cloud's cheapest candidate carries with the minima
(TaskMin::rec, skyopt_step.cuh); the full evaluation and solve_kernel read it
from the candidate tables. The records of the fused step must equal, bit for
bit, those read from the tables (every field but the slot, see
_records_only): forced by the full evaluation, and by solve_kernel after
separate launches (scan mode fast-split). The suites hold GCP accelerator
slots (host plus accelerator price), us-first partitions, zone-split slots,
reserved-node prices and blocked lists."""
import numpy as np
import pytest

from skypilot_b200 import engine
from skypilot_b200 import workloads
from tests import reservation_runner
from tests import reservation_scenarios
from tests import scenario_runner as runner
from tests import scenarios
from tests.test_gpu_chain_handoff import _state

pytestmark = pytest.mark.gpu


def _records(monkeypatch, suite, mode, path=None):
    """Per chain scenario of `suite`, run in scan mode `mode` on chain path
    `path`: every engine.solve call's chosen records, chosen indices, DAG
    results and kernel form, and what the scenario covers."""
    if suite == 'reservations':
        catalog = reservation_scenarios.CATALOG
        cases = reservation_runner.optimizer_scenarios()
    elif suite == 'regfilter':
        catalog = scenarios.CATALOGS['regfilter']
        cases = scenarios.EXTRA_GOLDEN_SUITES['regfilter']()
    else:
        catalog = scenarios.CATALOGS[suite]
        cases = scenarios.ALL_SUITES[suite]()
    store = runner.activate_catalog(catalog)
    calls = []
    real = engine.solve

    def solve(builder, *args, **kwargs):
        sol = real(builder, *args, **kwargs)
        n = sol.packed.n_tasks
        calls.append({
            'form': int(sol.stats.scan_form),
            'dag': [[int(d['status']), int(d['task_fail']),
                     float(d['objective']).hex()]
                    for d in sol.dag[:sol.packed.n_dags]],
            'index': sol.chosen_index[:n].tolist(),
            'chosen': [[int(c['slot']), int(c['inst_id']), int(c['region_id']),
                        int(c['zone_id']), float(c['hourly']).hex(),
                        float(c['value']).hex()] for c in sol.chosen[:n]],
        })
        return sol

    out = {}
    with monkeypatch.context() as m, runner.forced_paths(store, mode=mode,
                                                         chain=path):
        m.setattr(engine, 'solve', solve)
        for sc in cases:
            calls.clear()
            if suite == 'reservations':
                inner = {k: v for k, v in sc.items() if k != 'config'}
                with reservation_runner.inventory_of(sc):
                    rec = runner.run_scenario(inner, with_candidates=False)
            else:
                rec = runner.run_scenario(sc, with_candidates=False)
            if not rec.get('is_chain') or 'plan' not in rec:
                continue
            out[sc['name']] = {
                'calls': list(calls),
                'plan': rec['plan'],
                'reserved': bool(sc.get('reservations')),
            }
    return out


def _records_only(got):
    """Per scenario and call: the DAG results and every field of the chosen
    records but the slot. An any-of set can list one launchable in two of
    its slots, and which of those equal candidates a path picks (its slot
    and table index) is not part of the plan: the full evaluation takes the
    first in the table, the minima the first of the cheapest slot."""
    return {name: [(c['dag'], [ch[1:] for ch in c['chosen']])
                   for c in r['calls']] for name, r in got.items()}


@pytest.mark.parametrize('suite',
                         ['multi6k', 'fuzz6k', 'reservations', 'regfilter'])
def test_fused_records_equal_the_tables(suite, monkeypatch):
    fused = _records(monkeypatch, suite, 'auto')
    full = _records(monkeypatch, suite, 'auto', path='8')
    split = _records(monkeypatch, suite, 'fast-split')
    assert fused, 'no chain scenario ran'
    forms = {c['form'] for r in fused.values() for c in r['calls']}
    assert 4 in forms, forms
    assert 3 in {c['form'] for r in split.values() for c in r['calls']}
    want = _records_only(fused)
    assert want == _records_only(full)
    assert want == _records_only(split)
    # (a request with ordered resources can make calls that place nothing
    # before the one that does)
    placed = [c for r in fused.values() for c in r['calls']
              if all(d[0] == 0 for d in c['dag'])]
    assert placed
    assert all(ch[0] >= 0 for c in placed for ch in c['chosen'])
    plans = [p for r in fused.values() for p in r['plan']]
    if suite in ('multi6k', 'fuzz6k'):
        assert any(p['cloud'] == 'gcp' and p['accelerators'] for p in plans)
        assert any(p['zone'] for p in plans)
        assert any((p['region'] or '').startswith('us-') for p in plans)
    if suite == 'reservations':
        assert any(r['reserved'] for r in fused.values())


def _records_of(sol, n):
    c = sol.chosen[:n]
    d = sol.dag[0]
    return (int(d['status']), float(d['objective']).hex(),
            sol.chosen_index[:n].tolist(),
            [(int(x['slot']), int(x['inst_id']), int(x['region_id']),
              int(x['zone_id']), float(x['hourly']).hex(),
              float(x['value']).hex()) for x in c])


def test_device_resident_loop_keeps_the_records():
    """Fifty launches of the device-resident loop (the chain block no longer
    waits for the tables before its records; the hand-off word must still be
    re-armed each launch) give the records of a single call."""
    store = runner.activate_catalog(scenarios.CATALOGS['multi6k'])
    sc = workloads.chain('loop', [{'accelerators': 'V100', 'outputs_gb': 300},
                                  {'cpus': '8+', 'outputs_gb': 20},
                                  {'accelerators': 'A100:8', 'outputs_gb': 2500},
                                  {'accelerators': 'T4'}])
    one = engine.ProblemBuilder(store)
    dag, _ = workloads.build_dag(sc)
    _state(dag, one)
    want = _records_of(engine.solve(one), 4)
    assert want[0] == 0
    loop = engine.ProblemBuilder(store)
    dag, _ = workloads.build_dag(sc)
    _state(dag, loop)
    sol, iter_ms, _ = engine.solve_timed(loop, 50, False)
    assert len(iter_ms) == 50 and np.all(iter_ms > 0)
    assert int(sol.stats.scan_form) == 4
    assert _records_of(sol, 4) == want
