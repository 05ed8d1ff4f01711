"""A call's temporaries (the scan's list and fuzzy tables, a listing's arrays,
a non-quiet optimize's candidate tables) live in its context's scratch
buffer, which grows and is reused across calls of any size on one store.
Every repeated call must give what the first call of its shape gave, and a
call that fails with an argument error must leave the context usable."""
import ctypes

import pytest

import skypilot_b200 as sky
from skypilot_b200 import _native
from skypilot_b200 import engine
from skypilot_b200 import workloads
from tests import scenario_runner as runner
from tests import scenarios

pytestmark = pytest.mark.gpu

# multi6k has five AWS instance types with one T4 and four Lambda types
# with eight A100-80GB
_ACCS = [('aws', 'T4', 1), ('aws', 'A10G', 1), ('lambda', 'A100-80GB', 8),
         ('azure', 'T4', 1), ('gcp', 'T4', 4), ('aws', 'NoSuch', 1)]


def _scan(store, cap):
    """Argmin, instance list and fuzzy table of every query in _ACCS."""
    b = engine.ProblemBuilder(store)
    for cloud, acc, count in _ACCS:
        b.add_query(b.accelerator_query(cloud, acc, count, want_list=True,
                                        want_fuzzy=True))
    return engine.scan(b, list_cap=cap, fuzzy_cap=cap)


def _fields(a):
    """The bytes of every field of a record array (not its padding)."""
    return tuple(a[f].tobytes() for f in a.dtype.names)


def _scan_result(out):
    """Per-query results with their counts, and the list and fuzzy entries
    within the counts (a row's tail past its count is not written)."""
    r = out.results
    rows = []
    for q in range(len(r)):
        nl, nf = int(r['n_list'][q]), int(r['n_fuzzy'][q])
        rows.append((out.list_ids[q, :nl].tobytes(),
                     out.list_prices[q, :nl].tobytes(),
                     out.fuzzy_keys[q, :nf].tobytes(),
                     out.fuzzy_prices[q, :nf].tobytes()))
    return _fields(r), rows


def _listing():
    # repr: the listed prices may be NaN
    return repr(sky.catalog.list_accelerators(all_regions=True))


@pytest.fixture(name='solves')
def _solves(monkeypatch):
    """(builder, Solution) of every engine.solve the optimizer makes."""
    calls = []
    solve = engine.solve

    def recording(builder, *args, **kwargs):
        sol = solve(builder, *args, **kwargs)
        calls.append((builder, sol))
        return sol

    monkeypatch.setattr(engine, 'solve', recording)
    return calls


def _tables(sol):
    """Candidate counts, offsets, the ordered tables with their values, and
    the plan."""
    n = int(sol.table_offsets[-1])
    return (sol.task_n.tobytes(), sol.table_offsets.tobytes(),
            _fields(sol.tables[:n]), _fields(sol.chosen), _fields(sol.dag))


def test_scratch_is_reused_across_call_sizes(solves):
    store = runner.activate_catalog(scenarios.CATALOGS['multi6k'])
    outs = [_scan(store, cap) for cap in (2048, 1, 2048, 1)]
    # the large tables hold more than the small ones can
    assert outs[0].results['n_list'].max() >= 4
    assert outs[1].results['n_list'].max() == 1
    assert outs[1].results['n_fuzzy'].max() <= 1
    scans = [_scan_result(out) for out in outs]
    assert scans[2] == scans[0]
    assert scans[3] == scans[1]
    listing = _listing()
    assert len(listing) > 100 and _listing() == listing

    chain, _ = workloads.build_dag(workloads.chain_scenario(40))
    one, _ = workloads.build_dag(workloads.single('one_v100',
                                                  accelerators='V100'))
    for dag in (chain, one, chain, one):
        sky.Optimizer.optimize(dag, quiet=False)
    got = [_tables(sol) for _, sol in solves]
    assert len(got) == 4
    assert got[2] == got[0]
    assert got[3] == got[1]
    assert int(solves[0][1].table_offsets[-1]) > int(
        solves[1][1].table_offsets[-1])
    # the scan after the candidate tables still reads its own tables
    assert _scan_result(_scan(store, 2048)) == scans[0]


def test_failed_call_leaves_the_context_usable(solves):
    """A candidate capacity one entry short: skyopt_optimize fails with
    SKYOPT_ELIMIT in the copy-back; the next call on the store returns the
    tables of the call before the failure."""
    runner.activate_catalog(scenarios.CATALOGS['multi6k'])
    chain, _ = workloads.build_dag(workloads.chain_scenario(40))
    sky.Optimizer.optimize(chain, quiet=False)
    builder, first = solves[-1]
    want = _tables(first)
    n = int(first.table_offsets[-1])
    assert n > 1

    packed = builder.pack()
    short = engine.Solution(packed, True, table_cap=n - 1)
    csol = short.c_solution()
    lib = _native.load()
    prob = packed.c_problem()
    rc = lib.skyopt_optimize_blocks(builder.store.handle(0),
                                    ctypes.byref(prob), *packed.c_blocks(),
                                    ctypes.byref(csol),
                                    ctypes.byref(short.stats))
    assert rc == -4  # SKYOPT_ELIMIT
    assert b'candidate table needs' in lib.skyopt_last_error()

    assert _tables(engine.solve(builder, want_tables=True)) == want
    sky.Optimizer.optimize(chain, quiet=False)
    assert _tables(solves[-1][1]) == want
