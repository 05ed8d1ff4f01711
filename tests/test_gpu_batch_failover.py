"""Many DAGs failing over at once, on the device: optimize_batch with a
blocked list per DAG, and a batch session that re-solves only the DAGs whose
list changed, against one Optimizer.optimize per DAG with that DAG's list --
in every kernel mode and on every chain-DP path -- and
the argument checks of skyopt_session_resolve_dags."""
import ctypes

import numpy as np
import pytest

import skypilot_b200 as sky
from skypilot_b200 import _native
from skypilot_b200 import engine
from skypilot_b200 import optimizer as opt_lib
from skypilot_b200 import reservations
from skypilot_b200 import skypilot_config
from tests import reservation_scenarios
from tests import scenario_runner as runner
from tests import scenarios

pytestmark = pytest.mark.gpu
MODES = ['auto', 'fast-split', 'fast-noprune', 'queue', 'tile']


def _outcome(o, tasks):
    """A DAG's plan (records and per-task hourly cost), or its error text."""
    if isinstance(o, BaseException):
        return ('error', type(o).__name__, str(o))
    return [(runner.res_record(t.best_resources),
             t.best_resources.get_cost(3600)) for t in tasks]


def _single(spec, blocked):
    """A fresh Optimizer.optimize of `spec` under `blocked`."""
    dag, tasks = runner.build_dag(spec)
    try:
        sky.Optimizer.optimize(dag, blocked_resources=blocked or None,
                               quiet=True)
    except sky.exceptions.ResourcesUnavailableError as e:
        return _outcome(e, tasks)
    return _outcome(dag, tasks)


# ---- optimize_batch with per-DAG lists --------------------------------------
def check_fixture_lists(devices):
    """The blocked-list scenarios of the reference fixtures, each under its
    own list, batched with DAGs without a list and with a neighbour's list."""
    runner.activate_catalog(scenarios.CATALOGS['multi6k'])
    basic = [s for s in scenarios.basic_scenarios()
             if s.get('minimize', 'cost') == 'cost' and 'config' not in s]
    with_lists = [s for s in basic if s.get('blocked')]
    assert len(with_lists) >= 4
    plain = [s for s in basic if not s.get('blocked')][:24]
    specs, lists = [], []
    for k, s in enumerate(with_lists + plain):
        specs.append(s)
        own = runner.blocked_list(s) or []
        lists.append(own if s.get('blocked') else
                     (runner.blocked_list(with_lists[k % len(with_lists)])
                      if k % 3 == 0 else []))
    built = [runner.build_dag(s) for s in specs]
    out = sky.optimize_batch([d for d, _ in built], devices=devices,
                             blocked_resources_per_dag=lists,
                             return_exceptions=True)
    got = [_outcome(o, tasks) for o, (_, tasks) in zip(out, built)]
    want = [_single(s, bl) for s, bl in zip(specs, lists)]
    for k, (g, w) in enumerate(zip(got, want)):
        assert g == w, specs[k]['name']
    assert any(isinstance(o, Exception) for o in out)


def _cfg5_specs(n, seed=4):
    """cfg5-style single-task requests (tools/bench_batch.py's mix)."""
    rng = np.random.default_rng(seed)
    accs = [None, 'V100', 'T4', 'A100:8', 'L4', 'H100:8', 'A10G', 'K80',
            'A100', 'T4:4', 'V100:4', 'L4:8']
    regions = [None] * 10 + ['us-east-1', 'us-west-2']
    specs = []
    for k in range(n):
        res = {}
        acc = accs[int(rng.integers(len(accs)))]
        if acc:
            res['accelerators'] = acc
        cpus = [None, '2+', '8+', '32+'][int(rng.integers(4))]
        if cpus:
            res['cpus'] = cpus
        mem = [None, '16+', '4x'][int(rng.integers(3))]
        if mem and not acc:
            res['memory'] = mem
        if rng.uniform() < 0.5:
            res['use_spot'] = True
        region = regions[int(rng.integers(len(regions)))]
        if region:
            res['infra'] = f'aws/{region}'
        specs.append({'name': f'cfg5_{k}', 'tasks': [{'resources': [res]}]})
    return specs


_WILD_KINDS = ('zone', 'region', 'instance_type', 'cloud')


def _wildcard(rec, kind):
    """The blocked wildcard a failed launch of `rec` adds, of one kind."""
    w = {'cloud': rec['cloud'], 'use_spot': rec['use_spot']}
    if kind == 'zone' and rec['zone'] is not None:
        w['zone'] = rec['zone']
    elif kind in ('zone', 'region'):
        w['region'] = rec['region']
    elif kind == 'instance_type':
        w['instance_type'] = rec['instance_type']
    return w


_CFG5 = {}


def _cfg5_case(n=2000):
    """Seeded requests and per-DAG lists blocking their unblocked plans with
    wildcards of every kind (some lists empty), with the one-by-one
    outcomes; computed once per process."""
    if 'case' not in _CFG5:
        specs = _cfg5_specs(n)
        built = [runner.build_dag(s) for s in specs]
        out = sky.optimize_batch([d for d, _ in built], return_exceptions=True)
        rng = np.random.default_rng(17)
        lists = []
        for o, (_, tasks) in zip(out, built):
            r = int(rng.integers(6))
            if isinstance(o, Exception) or r >= 4:
                lists.append([])
                continue
            rec = runner.res_record(tasks[0].best_resources)
            lists.append(runner.blocked_list(
                {'blocked': [_wildcard(rec, _WILD_KINDS[r])]}))
        want = [_single(s, bl) for s, bl in zip(specs, lists)]
        _CFG5['case'] = (specs, lists, want)
    return _CFG5['case']


def check_cfg5(devices):
    runner.activate_catalog(scenarios.CATALOGS['multi50k'])
    specs, lists, want = _cfg5_case()
    built = [runner.build_dag(s) for s in specs]
    out = sky.optimize_batch([d for d, _ in built], devices=devices,
                             blocked_resources_per_dag=lists,
                             return_exceptions=True)
    got = [_outcome(o, tasks) for o, (_, tasks) in zip(out, built)]
    bad = [k for k in range(len(specs)) if got[k] != want[k]]
    assert not bad, (len(bad), got[bad[0]], want[bad[0]])
    assert sum(bool(bl) for bl in lists) > len(lists) // 3


# ---- the batch session -------------------------------------------------------
def _session_specs():
    by_name = {s['name']: s for s in scenarios.basic_scenarios()}
    resv = next(s for s in reservation_scenarios.reservation_scenarios()
                if s['name'] == 'aws_prio_v100_n4')
    big = next(s for s in scenarios.big_dag_scenarios()
               if s['name'] == 'sparse18')
    names = ['acc_V100', 'cpu_8p', 'acc_T4', 'spot_v100', 'acc_A100x8',
             'cfg2_chain8', 'chain3_mixed', 'cfg3_diamond', 'ordered_list',
             'chain_blocked_all']
    specs = [by_name[n] for n in names] + [big, resv]
    assert len(big['tasks']) == 18
    return specs, resv


def _device_ids(bs):
    """Global ids of the DAGs each shard's last resolve listed."""
    ids = set()
    for session, shard in zip(bs._sessions, bs._batch.shards):  # pylint: disable=protected-access
        if session is not None and session.last_dag_ids is not None:
            ids.update(shard[d] for d in session.last_dag_ids)
    return ids


def check_failover_rounds(devices):
    runner.activate_catalog(reservation_scenarios.CATALOG)
    specs, resv = _session_specs()
    ordered = {k for k, s in enumerate(specs) if s['name'] == 'ordered_list'}
    skypilot_config.set_config(resv['config'])
    reservations.set_reservations(resv['reservations'])
    try:
        built = [runner.build_dag(s) for s in specs]
        dags = [d for d, _ in built]
        rng = np.random.default_rng(23)
        # wildcard specs, rebuilt every round; chain_blocked_all starts
        # with its fixture list, which leaves it without a candidate
        wild = [list(s.get('blocked', [])) for s in specs]
        changed = set(range(len(specs)))
        exhausted = 0
        with sky.Optimizer.batch_session(dags, devices=devices) as bs:
            for rnd in range(6):
                lists = [runner.blocked_list({'blocked': w}) or []
                         for w in wild]
                out = bs.optimize(lists, return_exceptions=True)
                if rnd:
                    assert _device_ids(bs) == changed - ordered, rnd
                for k, (o, (_, tasks)) in enumerate(zip(out, built)):
                    assert _outcome(o, tasks) == _single(specs[k], lists[k]), (
                        rnd, specs[k]['name'])
                exhausted = sum(isinstance(o, Exception) for o in out)
                live = [k for k, o in enumerate(out)
                        if not isinstance(o, Exception)]
                picks = rng.choice(live, size=min(4, len(live)),
                                   replace=False)
                changed = set()
                for k in picks:
                    k = int(k)
                    tasks = built[k][1]
                    rec = runner.res_record(
                        tasks[int(rng.integers(len(tasks)))].best_resources)
                    wild[k].append(_wildcard(rec,
                                             _WILD_KINDS[(rnd + k) % 4]))
                    changed.add(k)
            assert exhausted >= 1
            # an unchanged call lists nothing and changes nothing
            lists = [runner.blocked_list({'blocked': w}) or [] for w in wild]
            first = bs.optimize(lists, return_exceptions=True)
            again = bs.optimize(
                [runner.blocked_list({'blocked': w}) or [] for w in wild],
                return_exceptions=True)
            assert _device_ids(bs) == set()
            assert [_outcome(o, t) for o, (_, t) in zip(first, built)] == [
                _outcome(o, t) for o, (_, t) in zip(again, built)]
            with pytest.raises(sky.exceptions.ResourcesUnavailableError):
                bs.optimize(lists)
            # a changed inventory: every DAG is stated and solved again
            before = list(bs._sessions)  # pylint: disable=protected-access
            reservations.set_reservations(resv['reservations'][1:])
            out = bs.optimize(lists, return_exceptions=True)
            assert not any(a is b for a, b in zip(before, bs._sessions)  # pylint: disable=protected-access
                           if a is not None)
            for k, (o, (_, tasks)) in enumerate(zip(out, built)):
                assert _outcome(o, tasks) == _single(specs[k], lists[k])
            # a reloaded catalog: the resident candidates mean nothing now
            runner.activate_catalog(scenarios.CATALOGS['three4k'])
            try:
                with pytest.raises(RuntimeError, match='catalog changed'):
                    bs.optimize(lists)
            finally:
                runner.activate_catalog(reservation_scenarios.CATALOG)
    finally:
        reservations.set_reservations(None)
        skypilot_config.set_config(None)


def run_all(devices=(0,)):
    devices = list(devices)
    check_fixture_lists(devices)
    check_cfg5(devices)
    check_failover_rounds(devices)


@pytest.mark.parametrize('mode', MODES)
def test_batch_and_session_in_every_kernel_mode(mode):
    stores = [runner.activate_catalog(scenarios.CATALOGS[name])
              for name in ('multi6k', 'multi50k')]
    with runner.forced_paths(*stores, mode=mode):
        run_all([0])
        run_all([0, 0])


@pytest.mark.parametrize('path', ['8', '32'])
def test_batch_and_session_on_every_chain_path(path):
    """The chain DP's full evaluation; the chain on the block that places
    the last task (runner.CHAIN_PATHS)."""
    with runner.forced_paths(chain=path):
        run_all([0])


# ---- skyopt_session_resolve_dags argument checks ---------------------------
def test_resolve_dags_rejects_bad_arguments():
    runner.activate_catalog(scenarios.CATALOGS['multi6k'])
    specs = [s for s in scenarios.basic_scenarios()
             if s['name'] in ('acc_V100', 'cpu_8p', 'cfg2_chain8')]
    dags = [runner.build_dag(s)[0] for s in specs]
    batch = opt_lib._Batch(dags, True, [0], [[]] * len(dags))  # pylint: disable=protected-access
    session = engine.Session(batch.builders[0])
    try:
        lib = _native.load()
        first = session.solution
        blocked = np.zeros(2, dtype=_native.BLOCKED_DTYPE)
        blocked[:] = -1
        n = len(dags)

        def call(ids, ranges, n_listed=None):
            ids = np.asarray(ids or [0], dtype=np.int32)
            spans = np.asarray(ranges or [(0, 0)], dtype=np.int32)
            sol = engine.Solution(session.packed, False)
            csol = sol.c_solution()
            return lib.skyopt_session_resolve_dags(
                session._handle, blocked.ctypes.data, 2, ids.ctypes.data,  # pylint: disable=protected-access
                spans.ctypes.data,
                len(ranges) if n_listed is None else n_listed,
                ctypes.byref(csol), None), sol

        for ids, ranges, n_listed in [([n], [(0, 0)], None),
                                      ([-1], [(0, 0)], None),
                                      ([1, 1], [(0, 0), (0, 1)], None),
                                      ([0], [(-1, 0)], None),
                                      ([0], [(0, 3)], None),
                                      ([0], [(2, 1)], None),
                                      ([0], [(0, 0)], -1)]:
            code, _ = call(ids, ranges, n_listed)
            assert code == -1, (ids, ranges, n_listed)  # SKYOPT_EINVAL
            assert lib.skyopt_last_error()
        # nothing listed: nothing launched, the previous plan comes back
        sol = session.resolve_dags([], [], [])
        assert sol.stats.total_launches == 0
        assert (sol.chosen_index[:first.packed.n_tasks] ==
                first.chosen_index[:first.packed.n_tasks]).all()
        assert (sol.dag['objective'] == first.dag['objective']).all()
        # listing one DAG under an empty range gives its first plan again
        sol = session.resolve_dags([], [1], [(0, 0)])
        assert sol.stats.total_launches == 2
        assert (sol.dag['objective'] == first.dag['objective']).all()
    finally:
        session.close()
