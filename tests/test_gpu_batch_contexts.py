"""Placement contexts on the device: one batch whose DAGs each carry their own
enabled clouds, SkyPilot config, reservation inventory and objective, against
the unmodified reference's records (tests/golden/reservations.json,
tests/golden/regfilter.json) and against one Optimizer.optimize per DAG under
the process state set to its context -- in every kernel mode, on every
chain-DP path, on one shard and on two -- plus per-context
reservation blocks that price the same (cloud, instance type, zone)
differently in one launch, the refusal of bad ranges, and a batch session's
failover rounds."""
import copy
import ctypes

import numpy as np
import pytest

import skypilot_b200 as sky
from skypilot_b200 import _native
from skypilot_b200 import engine
from skypilot_b200 import optimizer as opt_lib
from tests import reservation_runner
from tests import reservation_scenarios
from tests import scenario_runner as runner
from tests import scenarios
from tests import test_gpu_batch_failover as failover
from tests.test_batch_contexts import process_state

pytestmark = pytest.mark.gpu
MODES = ['auto', 'fast-split', 'fast-noprune', 'queue', 'tile']
INV = reservation_scenarios.RESERVATION_INVENTORY
AWS_PRIO = {'aws': {'prioritize_reservations': True}}
GCP_PRIO = {'gcp': {'prioritize_reservations': True}}
BOTH_PRIO = {'aws': {'prioritize_reservations': True},
             'gcp': {'prioritize_reservations': True}}
PROXY = {'aws': {'ssh_proxy_command': {'us-east-2': 'ssh -W %h:%p a',
                                       'eu-west-1': 'ssh -W %h:%p b',
                                       'us-west-2': 'ssh -W %h:%p c'}}}


def _target(spec):
    return (sky.OptimizeTarget.TIME if spec.get('minimize') == 'time' else
            sky.OptimizeTarget.COST)


def _context_of(spec):
    """A fixture scenario's config and inventory as a context of its own."""
    return sky.PlacementContext(config=spec.get('config') or {},
                                reservations=spec.get('reservations') or [],
                                minimize=_target(spec))


def _error(e):
    return {'type': type(e).__name__, 'message': str(e)}


def batch_records(specs, contexts, devices):
    """Every DAG of one batch: plan (optimize_batch), ordered candidate
    tables and DP objective (the same batch's device problem with tables),
    or the error, in the records' layout. A request the reference refuses
    while it is constructed (ValueError) is left out of the batch."""
    records, built, kept = {}, [], []
    for k, s in enumerate(specs):
        try:
            built.append(runner.build_dag(s))
            kept.append(k)
        except ValueError as e:
            records[k] = {'name': s['name'], 'error': _error(e)}
    specs = [specs[k] for k in kept]
    contexts = [contexts[k] for k in kept]
    dags = [d for d, _ in built]
    lists = [runner.blocked_list(s) or [] for s in specs]
    out = sky.optimize_batch(dags, devices=devices, return_exceptions=True,
                             blocked_resources_per_dag=lists,
                             contexts=contexts)
    batch = opt_lib._Batch(dags, True, devices, lists, contexts=contexts)  # pylint: disable=protected-access
    sols = [engine.solve(b, device=dev, want_tables=True) if b.dags else None
            for b, dev in zip(batch.builders, devices)]
    for i, (spec, (_, tasks)) in enumerate(zip(specs, built)):
        rec = records[kept[i]] = {'name': spec['name']}
        if isinstance(out[i], BaseException):
            rec['error'] = _error(out[i])
            continue
        rec['plan'] = [runner.res_record(t.best_resources) for t in tasks]
        k = i % len(devices)
        d = batch.shards[k].index(i)
        sol, problem = sols[k], batch.problems[i]
        first = batch.first_task[i]
        rec['candidates'] = []
        for j in range(len(tasks)):
            rows = []
            for cand in sol.task_table(first + j):
                r = problem.launchable(cand)
                rows.append([str(r.cloud).lower(), r.instance_type, r.region,
                             r.zone, float(cand['value'])])
            rec['candidates'].append(rows)
        rec['objective'] = float(sol.dag[d]['objective'])
    return [records[k] for k in sorted(records)]


# ---- 1. reference parity ----------------------------------------------------
def check_reservation_fixture(devices):
    payload = reservation_runner.golden()
    gold = {r['name']: r for r in payload['records']}
    runner.activate_catalog(payload['catalog'])
    specs = reservation_runner.optimizer_scenarios()
    got = batch_records(specs, [_context_of(s) for s in specs], devices)
    bad = []
    for spec, rec in zip(specs, got):
        g = gold[spec['name']]
        if 'error' in g or 'error' in rec:
            if g.get('error') != rec.get('error'):
                bad.append((spec['name'], 'error'))
            continue
        if rec['candidates'] != g['candidates']:
            bad.append((spec['name'], 'candidates'))
        if rec['plan'] != g['plan']:
            bad.append((spec['name'], 'plan', g['plan'], rec['plan']))
        if (rec['objective'] != g['objective'] if g['is_chain'] else
                not runner.close(g['objective'], rec['objective'])):
            bad.append((spec['name'], 'objective'))
    assert not bad, bad


def check_regfilter_fixture(devices):
    payload = runner.load_golden('regfilter')
    gold = {r['name']: r for r in payload['records']}
    runner.activate_catalog(payload['catalog'])
    specs = scenarios.region_filter_scenarios()
    got = batch_records(specs, [_context_of(s) for s in specs], devices)
    bad = []
    for spec, rec in zip(specs, got):
        # the reference's record, as its own suite compares it
        # (test_gpu_region_filter.py), and the single-DAG path bit for bit
        diffs = runner.compare(gold[spec['name']], rec)
        if diffs:
            bad.append((spec['name'], diffs[:2]))
        alone = runner.run_scenario(spec)
        for key in ('error', 'candidates', 'plan'):
            if alone.get(key) != rec.get(key):
                bad.append((spec['name'], key))
    assert not bad, bad


# ---- 2. self-consistency at scale ------------------------------------------
def _scale_contexts():
    more = copy.deepcopy(INV)
    for r in more:
        r['available'] += 2
    fewer = [dict(r, available=1) for r in INV]
    t = sky.OptimizeTarget
    return [
        None,
        sky.PlacementContext(enabled_clouds=['aws'], config=AWS_PRIO,
                             reservations=INV),
        sky.PlacementContext(enabled_clouds=['aws', 'gcp'], config=BOTH_PRIO,
                             reservations=more, minimize=t.TIME),
        sky.PlacementContext(enabled_clouds=['gcp', 'azure'],
                             config=GCP_PRIO, reservations=INV),
        sky.PlacementContext(enabled_clouds=[]),
        sky.PlacementContext(config=PROXY, reservations=[]),
        sky.PlacementContext(config=BOTH_PRIO, reservations=fewer),
        # the first context's config, another inventory and objective
        sky.PlacementContext(enabled_clouds=['aws', 'gcp'],
                             config=copy.deepcopy(AWS_PRIO),
                             reservations=more[:2], minimize=t.TIME),
    ]


def _scale_specs(n=2000):
    by_name = {s['name']: s for s in scenarios.basic_scenarios()}
    big = next(s for s in scenarios.big_dag_scenarios()
               if s['name'] == 'sparse18')
    shaped = [by_name[n] for n in ('cfg2_chain8', 'chain3_mixed',
                                   'cfg3_diamond', 'ordered_list')]
    specs = failover._cfg5_specs(n - 20, seed=9)  # pylint: disable=protected-access
    for k in range(20):
        specs.insert(97 * k + 5, dict(shaped[k % 4], name=f'shaped_{k}'))
    ctxs = _scale_contexts()
    contexts = [ctxs[k % len(ctxs)] for k in range(len(specs))]
    # the general DAG beyond the device enumeration: COST contexts only
    # (TIME has no exact search for it)
    for k in (3, 11, 19):
        specs.insert(k * 90, dict(big, name=f'big_{k}'))
        contexts.insert(k * 90, ctxs[(1, 5, 6)[k % 3]])
    return specs, contexts


def _single(spec, ctx, blocked=None):
    """One Optimizer.optimize of `spec` with the process state set to
    `ctx`."""
    dag, tasks = runner.build_dag(spec)
    target = (ctx.minimize if ctx is not None and ctx.minimize is not None
              else sky.OptimizeTarget.COST)
    with process_state(ctx):
        try:
            sky.Optimizer.optimize(dag, target, blocked or None, quiet=True)
        except (sky.exceptions.ResourcesUnavailableError,
                sky.exceptions.NoCloudAccessError) as e:
            return failover._outcome(e, tasks)  # pylint: disable=protected-access
    return failover._outcome(dag, tasks)  # pylint: disable=protected-access


_SCALE = {}


def check_scale(devices):
    runner.activate_catalog(reservation_scenarios.CATALOG)
    if 'case' not in _SCALE:
        specs, contexts = _scale_specs()
        _SCALE['case'] = (specs, contexts,
                          [_single(s, c) for s, c in zip(specs, contexts)])
    specs, contexts, want = _SCALE['case']
    built = [runner.build_dag(s) for s in specs]
    out = sky.optimize_batch([d for d, _ in built], devices=devices,
                             contexts=contexts, return_exceptions=True)
    got = [failover._outcome(o, t) for o, (_, t) in zip(out, built)]  # pylint: disable=protected-access
    bad = [k for k in range(len(specs)) if got[k] != want[k]]
    assert not bad, (len(bad), specs[bad[0]]['name'], got[bad[0]],
                     want[bad[0]])
    kinds = {type(o).__name__ for o in out if isinstance(o, Exception)}
    assert 'NoCloudAccessError' in kinds


# ---- 3. one (cloud, instance type, zone), two counts, one launch ----------
def check_crafted(devices):
    store = runner.activate_catalog(reservation_scenarios.CATALOG)
    rec = dict(cloud='aws', instance_type='p3.2xlarge', zone='us-west-2b',
               name='cr-shared', available=0)
    counts = [1, 3, 0, 6]
    contexts = [sky.PlacementContext(enabled_clouds=['aws'], config=AWS_PRIO,
                                     reservations=[dict(rec, available=c)])
                for c in counts]
    dags = []
    for _ in counts:
        with sky.Dag() as dag:
            sky.Task('t', num_nodes=4).set_resources(sky.Resources(
                infra='aws', instance_type='p3.2xlarge'))
        dags.append(dag)
    batch = opt_lib._Batch(dags, True, devices, [[]] * len(dags),  # pylint: disable=protected-access
                           contexts=contexts)
    assert len(batch.shards[0]) >= 2
    checked = 0
    for k, b in enumerate(batch.builders):
        if not b.dags:
            continue
        sol = engine.solve(b, device=devices[k], want_tables=True)
        assert sol.packed.n_reservations == len(
            {counts[i] for i in batch.shards[k]})
        for i in batch.shards[k]:
            rows = sol.task_table(batch.first_task[i])
            assert len(rows)
            for cand in rows:
                zone = batch.problems[i].launchable(cand).zone
                reserved = counts[i] if zone == rec['zone'] else 0
                want = (float(float(cand['hourly']) * 1.0) *
                        max(4 - reserved, 0))
                assert float(cand['value']) == want, (counts[i], zone)
                checked += zone == rec['zone']
    assert checked >= len(counts)
    # malformed ranges and block indices are refused before any launch
    b = batch.builders[0]
    lib = _native.load()
    for bad in ('descending', 'outside', 'block'):
        packed = b.pack()
        if bad == 'descending':
            packed.reservation_ranges[1] = packed.reservation_ranges[-1] + 1
            packed.reservation_ranges[-1] = 0
        elif bad == 'outside':
            packed.reservation_ranges[-1] = packed.n_reservations + 1
        else:
            packed.slots['pad_'][0] = len(packed.reservation_ranges)
        sol = engine.Solution(packed, False)
        code = lib.skyopt_optimize_blocks(
            store.handle(devices[0]), ctypes.byref(packed.c_problem()),
            *packed.c_blocks(), ctypes.byref(sol.c_solution()),
            ctypes.byref(sol.stats))
        assert code == -1, bad  # SKYOPT_EINVAL
        assert lib.skyopt_last_error()


# ---- 4. a batch session over mixed contexts ---------------------------------
def check_session(devices):
    runner.activate_catalog(reservation_scenarios.CATALOG)
    by_name = {s['name']: s for s in scenarios.basic_scenarios()}
    resv = [s for s in reservation_runner.optimizer_scenarios()
            if s['name'] in ('aws_prio_v100_n4', 'chain3_egress',
                             'diamond4', 'gcp_prio_v100_n3')]
    plain = [by_name[n] for n in ('acc_V100', 'cpu_8p', 'acc_T4',
                                  'spot_v100', 'cfg2_chain8', 'ordered_list')]
    ctxs = _scale_contexts()
    specs = resv + plain + resv
    contexts = ([_context_of(s) for s in resv] +
                [ctxs[k % len(ctxs)] for k in range(len(plain))] +
                [ctxs[1], ctxs[2], ctxs[6], ctxs[7]])
    ordered = {k for k, s in enumerate(specs) if s['name'] == 'ordered_list'}
    built = [runner.build_dag(s) for s in specs]
    rng = np.random.default_rng(31)
    wild = [list(s.get('blocked', [])) for s in specs]
    changed = set(range(len(specs)))
    with sky.Optimizer.batch_session([d for d, _ in built], devices=devices,
                                     contexts=contexts) as bs:
        for rnd in range(5):
            lists = [runner.blocked_list({'blocked': w}) or [] for w in wild]
            out = bs.optimize(lists, return_exceptions=True)
            if rnd:
                assert failover._device_ids(bs) == changed - ordered, rnd  # pylint: disable=protected-access
            for k, (o, (_, tasks)) in enumerate(zip(out, built)):
                assert failover._outcome(o, tasks) == _single(  # pylint: disable=protected-access
                    specs[k], contexts[k], lists[k]), (rnd, specs[k]['name'])
            live = [k for k, o in enumerate(out)
                    if not isinstance(o, Exception)]
            changed = set()
            for k in rng.choice(live, size=min(4, len(live)), replace=False):
                k = int(k)
                tasks = built[k][1]
                rec = runner.res_record(
                    tasks[int(rng.integers(len(tasks)))].best_resources)
                wild[k].append(failover._wildcard(  # pylint: disable=protected-access
                    rec, failover._WILD_KINDS[(rnd + k) % 4]))  # pylint: disable=protected-access
                changed.add(k)


def run_all(devices=(0,)):
    devices = list(devices)
    check_reservation_fixture(devices)
    check_regfilter_fixture(devices)
    check_scale(devices)
    check_crafted(devices)
    check_session(devices)


@pytest.mark.parametrize('mode', MODES)
def test_contexts_in_every_kernel_mode(mode):
    stores = [runner.activate_catalog(spec) for spec in (
        reservation_scenarios.CATALOG, scenarios.CATALOGS['regfilter'])]
    with runner.forced_paths(*stores, mode=mode):
        run_all([0])
        run_all([0, 0])


@pytest.mark.parametrize('path', ['8', '32'])
def test_contexts_on_every_chain_path(path):
    """The chain DP's full evaluation; the chain on the block that places
    the last task (runner.CHAIN_PATHS)."""
    with runner.forced_paths(chain=path):
        run_all([0])
