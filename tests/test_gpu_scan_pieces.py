"""The class-table scan's pieces: each group's share of the resident blocks
and the cut of its chunks, by estimated cost (the default) or by equal chunk
counts (engine.set_scan_pieces(equal=True)). Pieces only decide which block
prunes what, so both give the unpruned scan's results, in the fused step
(`auto`) and in separate launches (`fast-split`)."""
import contextlib

import numpy as np
import pytest

from skypilot_b200 import _native
from skypilot_b200 import engine
from skypilot_b200 import workloads
from tests import reservation_runner
from tests import scenario_runner as runner
from tests import scenarios
from tests.test_gpu_chain_handoff import _state
from tests.test_gpu_chain_lean import _flagship_outputs

pytestmark = pytest.mark.gpu

RUNS = [('auto', False), ('auto', True), ('fast-split', False),
        ('fast-split', True)]
RUN_IDS = [f'{mode}-{"equal" if eq else "weighted"}' for mode, eq in RUNS]


@contextlib.contextmanager
def _pieces(equal):
    try:
        engine.set_scan_pieces(equal=equal)
        yield
    finally:
        engine.set_scan_pieces()


def _cfg4_builder():
    store = runner.activate_catalog(workloads.CATALOGS['cfg4'])
    dag, _ = workloads.build_dag(workloads.chain_scenario(32))
    builder = engine.ProblemBuilder(store)
    _state(dag, builder)
    return store, builder


def _scan(store, builder, mode, equal):
    with _pieces(equal), runner.forced_paths(store, mode=mode):
        out = engine.scan(builder)
    return out.results['best_row'].copy(), out.results['any_stage1'].copy()


def test_scan_results_same_under_both_piece_plans():
    """skyopt_scan on the cfg4 chain's queries (every group wants
    any_stage1, as gate queries do): best rows and any_stage1 bits equal the
    unpruned scan's under both piece plans."""
    store, builder = _cfg4_builder()
    want = _scan(store, builder, 'fast-noprune', False)
    assert (want[0] >= 0).any() and want[1].any()
    for mode, equal in RUNS:
        got = _scan(store, builder, mode, equal)
        assert np.array_equal(got[0], want[0]), (mode, equal)
        assert np.array_equal(got[1], want[1]), (mode, equal)


@pytest.mark.parametrize('mode,equal', RUNS, ids=RUN_IDS)
def test_plans_same_under_both_piece_plans(mode, equal):
    """Plans and candidate tables of the multi6k, fuzz6k, reservation and
    region-filter suites match the reference's, and the cfg4 chain's outputs
    are bit-identical to the unpruned scan's."""
    with _pieces(equal):
        bad, _ = runner.check_chain_suites(mode)
        assert not bad, bad
        store = runner.activate_catalog(reservation_runner.golden()['catalog'])
        with runner.forced_paths(store, mode=mode):
            bad = reservation_runner.check_all()
        assert not bad, bad
        payload = runner.load_golden('regfilter')
        store = runner.activate_catalog(payload['catalog'])
        records = {r['name']: r for r in payload['records']}
        with runner.forced_paths(store, mode=mode):
            bad = [(sc['name'], d[:2])
                   for sc in scenarios.region_filter_scenarios()
                   for d in [runner.compare(records[sc['name']],
                                            runner.run_scenario(sc))] if d]
        assert not bad, bad
        got = _flagship_outputs('cfg4', mode=mode)
    want = _flagship_outputs('cfg4', mode='fast-noprune')
    for name, arr in want.items():
        assert arr.tobytes() == got[name].tobytes(), name


def _check_cover(plan, store):
    """Every group's pieces are consecutive in launch order and cover its
    cloud's chunks once, in order; at most one piece per block."""
    p = plan.pieces
    assert 0 < len(p) <= plan.grid
    offs = np.asarray(store.columns['cloud_row_offsets']) // _native.ZONE_ROWS
    groups = p['group']
    assert (np.diff(groups) >= 0).all()
    for g in np.unique(groups):
        mine = p[groups == g]
        c = int(mine['cloud'][0])
        assert (mine['cloud'] == c).all() and (mine['col'] == mine['col'][0]).all()
        assert mine['chunk_begin'][0] == offs[c]
        assert mine['chunk_end'][-1] == offs[c + 1]
        assert (mine['chunk_begin'] < mine['chunk_end']).all()
        assert (mine['chunk_begin'][1:] == mine['chunk_end'][:-1]).all()


def test_weighted_plan_covers_every_chunk_once():
    """The cost-weighted plan of the cfg4 chain, for the fused launch and the
    separate scan launch: full, ordered, disjoint cover, and the Lambda group
    (nearly every chunk passes its zone map) gets more, smaller pieces than
    under equal chunk counts."""
    store, builder = _cfg4_builder()
    lam = store.cloud_index['lambda']
    for fused in (True, False):
        weighted = engine.scan_pieces(builder, fused=fused)
        _check_cover(weighted, store)
        with _pieces(True):
            equal = engine.scan_pieces(builder, fused=fused)
        _check_cover(equal, store)
        n_w = int((weighted.pieces['cloud'] == lam).sum())
        n_e = int((equal.pieces['cloud'] == lam).sum())
        assert n_w > n_e, (fused, n_w, n_e)
        assert [list(q) for q in weighted.group_queries] == \
            [list(q) for q in equal.group_queries]
    lib = _native.load()
    assert lib.skyopt_set_scan_pieces(2) == -1
    assert b'unknown' in lib.skyopt_last_error()
