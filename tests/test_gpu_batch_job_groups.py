"""JobGroups on the device: `optimize_batch(..., job_groups=True)`,
`batch_session(..., job_groups=True)` and `Optimizer.optimize_job_group`
against a model that is the host algorithm optimize_job_group ran before the
selection moved into solve_kernel (`Optimizer._optimize_job_group_host`:
each job stated as a single-task DAG, candidate tables copied back, scores,
intersection and sums on the host), and every other DAG of the batch
against `Optimizer.optimize` -- in every kernel mode, on one shard and on
two, on every chain-DP path -- plus the SKYOPT_EINVAL
checks of the new DAG kind."""
import ctypes
import random

import pytest

import skypilot_b200 as sky
from skypilot_b200 import _native
from skypilot_b200 import engine
from skypilot_b200 import optimizer as opt_lib
from skypilot_b200 import placement_context
from skypilot_b200.dag import DagExecution
from tests import azmap_runner
from tests import azmap_scenarios
from tests import reservation_scenarios
from tests import scenario_runner as runner
from tests import scenarios

pytestmark = pytest.mark.gpu
MODES = ['auto', 'fast-split', 'fast-noprune', 'queue', 'tile']
COST, TIME = sky.OptimizeTarget.COST, sky.OptimizeTarget.TIME
_ERRORS = (sky.exceptions.ResourcesUnavailableError,
           sky.exceptions.NoCloudAccessError)


def _build(spec):
    dag, tasks = runner.build_dag(spec)
    dag.name = spec['name']
    if spec.get('kind') == 'job_group':
        dag.set_execution(DagExecution.PARALLEL)
    return dag, tasks


def _outcome(o, tasks):
    """Plan and resources (the override) of every task, or the error."""
    if isinstance(o, BaseException):
        return ('error', type(o).__name__, str(o))
    return [(runner.res_record(t.best_resources),
             sorted((str(r.cloud).lower(), r.region) for r in t.resources))
            for t in tasks]


def _model(spec, minimize=COST, blocked=None, ctx=None):
    """A fresh copy of `spec` placed by the host algorithm (JobGroups) or by
    Optimizer.optimize (every other DAG), under `ctx`."""
    dag, tasks = _build(spec)
    try:
        with placement_context.active(ctx):
            if spec.get('kind') == 'job_group':
                opt_lib.Optimizer._optimize_job_group_host(  # pylint: disable=protected-access
                    dag, minimize, list(blocked or []), quiet=True)
            else:
                sky.Optimizer.optimize(dag, minimize, blocked or None,
                                       quiet=True)
    except _ERRORS as e:
        return _outcome(e, tasks)
    return _outcome(dag, tasks)


def _batch(specs, devices, minimize=COST, lists=None, contexts=None):
    built = [_build(s) for s in specs]
    out = sky.Optimizer.optimize_batch(
        [d for d, _ in built], minimize, devices=devices,
        return_exceptions=True, blocked_resources_per_dag=lists,
        contexts=contexts, job_groups=True)
    return [_outcome(o, tasks) for o, (_, tasks) in zip(out, built)]


def _check(specs, devices, minimize=COST, lists=None, contexts=None):
    got = _batch(specs, devices, minimize, lists, contexts)
    for k, spec in enumerate(specs):
        ctx = None if contexts is None else contexts[k]
        want = _model(spec, ctx.minimize if ctx is not None and
                      ctx.minimize is not None else minimize,
                      None if lists is None else lists[k], ctx)
        assert got[k] == want, (spec['name'], got[k], want)
    return got


# ---- the recorded JobGroups -------------------------------------------------
def check_records(devices):
    """The jobgroup_multi6k, AZ-mapping and reservation JobGroups, each
    suite in one batch; where the reference is deterministic (one job, at
    most one common infra) also equal to its recorded plan and overrides."""
    payload = runner.load_golden('jobgroup_multi6k')
    runner.activate_catalog(dict(payload['catalog']))
    records = {r['name']: r for r in payload['records']}
    cases = scenarios.job_group_cases()
    for target in (COST, TIME):
        specs = [c for c in cases
                 if (c.get('minimize', 'cost') == 'cost') == (target == COST)]
        got = _check(specs, devices, target)
        for spec, g in zip(specs, got):
            rec = records[spec['name']]
            if 'error' in rec:
                assert g[2] == rec['error']['message']
            elif len(spec['tasks']) == 1 or len(rec['common_infras']) <= 1:
                if target == COST:
                    assert [p for p, _ in g] == rec['plan']
    azmap_runner.activate()
    _check(azmap_scenarios.job_group_cases(), devices)
    resv = [s for s in reservation_scenarios.reservation_scenarios()
            if s.get('kind') == 'job_group']
    assert resv
    runner.activate_catalog(dict(reservation_scenarios.CATALOG))
    for s in resv:
        ctx = placement_context.PlacementContext(
            config=s.get('config'), reservations=s.get('reservations'))
        _check([s], devices, contexts=[ctx])


# ---- seeded groups mixed with chains and general DAGs -----------------------
_ACCS = ['V100', 'T4', 'A100', 'A100:8', 'K80', 'V100:4', None, None]


def _job(rng, store, pin):
    spec = {}
    acc = rng.choice(_ACCS)
    if acc is None:
        spec['cpus'] = rng.choice(['4+', '8+', '16+'])
    else:
        spec['accelerators'] = acc
    if rng.random() < 0.2:
        spec['use_spot'] = True
    if pin is not None:
        cloud, region, zone = pin
        spec['cloud'] = cloud
        if region is not None:
            spec['region'] = region
        if zone is not None:
            spec['zone'] = zone
    if rng.random() < 0.3:
        spec['num_nodes'] = rng.randint(2, 4)
    if rng.random() < 0.15:
        spec['inputs'] = [rng.choice(['s3://b/x', 'gs://b/x']),
                          rng.choice([1.0, 50.0, 800.0])]
    del store
    return spec


def _pin(rng, store, level):
    table = rng.choice([t for t in store.clouds])
    if level == 'cloud':
        return (table.name, None, None)
    region = rng.choice(table.region_names)
    zones = [z for z in table.zone_names if z.startswith(region)]
    if level == 'zone' and zones:
        return (table.name, region, rng.choice(zones))
    return (table.name, region, None)


def random_group(rng, store, name):
    n = rng.choice([1, 1, 2, 2, 3, 4, 5, 8])
    if rng.random() < 0.03:
        n = 40
    shape = rng.choice(['free', 'free', 'cloud', 'region', 'zone', 'split',
                        'unavailable'])
    shared = _pin(rng, store, shape) if shape in (
        'cloud', 'region', 'zone') else None
    jobs = []
    for j in range(n):
        pin = shared
        if shape == 'split':
            pin = (store.clouds[j % len(store.clouds)].name, None, None)
        elif shape in ('region', 'zone') and rng.random() < 0.5:
            pin = None
        jobs.append(_job(rng, store, pin))
    if shape == 'unavailable':
        jobs[rng.randrange(n)] = {'accelerators': 'A100:3'}
    tasks = []
    for j, spec in enumerate(jobs):
        extra = {k: spec.pop(k) for k in ('num_nodes', 'inputs') if k in spec}
        tasks.append(dict(name=f'{name}_j{j}', resources=[spec], **extra))
    return dict(name=name, kind='job_group', tasks=tasks)


def mixed_specs(seed, n_groups):
    rng = random.Random(seed)
    store = runner.activate_catalog(scenarios.CATALOGS['multi6k'])
    basic = [s for s in scenarios.basic_scenarios()
             if s.get('minimize', 'cost') == 'cost' and 'config' not in s
             and not s.get('blocked')]
    specs = []
    for k in range(n_groups):
        specs.append(random_group(rng, store, f'g{seed}_{k}'))
        if k % 8 == 0:
            specs.append(dict(basic[(k // 8) % len(basic)],
                              name=f'd{seed}_{k}'))
    return specs


def check_mixed(devices, n_groups=1000, seed=3):
    """Seeded groups of 1-40 jobs (pinned clouds, regions and zones, spot,
    up to 4 nodes, inputs, groups without a common infra, a job that
    cannot be placed) with chains and general DAGs in one batch, a TIME
    context on every fifth DAG."""
    specs = mixed_specs(seed, n_groups)
    time_ctx = placement_context.PlacementContext(minimize=TIME)
    contexts = [time_ctx if k % 5 == 4 else None for k in range(len(specs))]
    got = _check(specs, devices, contexts=contexts)
    groups = [g for g, s in zip(got, specs) if s.get('kind') == 'job_group']
    errors = sum(g[0] == 'error' for g in groups)
    shared = sum(g[0] != 'error' and len({(p['cloud'], p['region'])
                                          for p, _ in g}) == 1 and len(g) > 1
                 for g in groups)
    fallback = sum(g[0] != 'error' and len({(p['cloud'], p['region'])
                                            for p, _ in g}) > 1
                   for g in groups)
    assert errors and shared and fallback, (errors, shared, fallback)


# ---- crafted ties -------------------------------------------------------------
def check_ties(devices):
    """Equal totals across infras (two equal jobs pinned to a cloud, whose
    regions repeat the synthetic prices) and equal scores inside an infra
    in different candidate order (spot jobs, one candidate per zone, next
    to region-level on-demand ones)."""
    store = runner.activate_catalog(scenarios.CATALOGS['multi6k'])
    specs = []
    for t in store.clouds:
        for acc in ('V100', 'T4', None):
            job = {'cloud': t.name}
            if acc is None:
                job['cpus'] = '8+'
            else:
                job['accelerators'] = acc
            spot = dict(job, use_spot=True)
            for tag, jobs in (('same', [job, dict(job)]),
                              ('spot', [spot, job, dict(spot)])):
                specs.append(dict(
                    name=f'tie_{tag}_{t.name}_{acc}', kind='job_group',
                    tasks=[dict(name=f'j{k}', resources=[r])
                           for k, r in enumerate(jobs)]))
    _check(specs, devices)
    _check(specs, devices, TIME)


def check_most_regions(devices):
    """The catalog with the most regions of the test suite."""
    store = runner.activate_catalog(scenarios.CATALOGS['fuzzmany'])
    rng = random.Random(11)
    _check([random_group(rng, store, f'many{k}') for k in range(150)],
           devices)


# ---- batch sessions ----------------------------------------------------------
def _session_model(specs, lists, contexts):
    return [_model(s, COST, lists[k], contexts[k])
            for k, s in enumerate(specs)]


def check_session(devices):
    """Five rounds that block each group's chosen region, until groups fall
    back (no common infra) and then error; each round equals the model on
    a fresh copy of the DAGs as opened. Round 4 passes new reservation
    inventories (a re-price), round 5 a new config (a full solve). The DAGs
    re-solved by a blocked-list round are those whose list changed."""
    runner.activate_catalog(dict(reservation_scenarios.CATALOG))
    rng = random.Random(5)
    store = sky.catalog.get_store()
    specs = [random_group(rng, store, f's{k}') for k in range(60)]
    specs += [s for s in reservation_scenarios.reservation_scenarios()
              if s.get('kind') == 'job_group']
    specs.append(dict(scenarios.basic_scenarios()[0], name='plain'))
    inventory = reservation_scenarios.RESERVATION_INVENTORY
    prio = {'aws': {'prioritize_reservations': True},
            'gcp': {'prioritize_reservations': True}}
    contexts = [placement_context.PlacementContext(config=prio,
                                                   reservations=inventory)
                for _ in specs]
    built = [_build(s) for s in specs]
    dags = [d for d, _ in built]
    lists = [[] for _ in specs]
    with sky.Optimizer.batch_session(dags, devices=devices, contexts=contexts,
                                     job_groups=True) as session:
        for rnd in range(6):
            if rnd == 4:
                contexts = [placement_context.PlacementContext(
                    config=prio, reservations=inventory[:3])
                            for _ in specs]
                out = session.optimize(lists, return_exceptions=True,
                                       contexts=contexts)
            elif rnd == 5:
                contexts = [placement_context.PlacementContext(
                    config={'aws': {'prioritize_reservations': False}},
                    reservations=inventory[:3]) for _ in specs]
                out = session.optimize(lists, return_exceptions=True,
                                       contexts=contexts)
            else:
                out = session.optimize(lists, return_exceptions=True)
            got = [_outcome(o, tasks) for o, (_, tasks) in zip(out, built)]
            assert got == _session_model(specs, lists, contexts), rnd
            changed = set()
            for k, (g, s) in enumerate(zip(got, specs)):
                if s.get('kind') != 'job_group' or g[0] == 'error':
                    continue
                # block the region of the first job, on its cloud
                cloud, region = g[0][0]['cloud'], g[0][0]['region']
                lists[k] = lists[k] + [runner.blocked_list(dict(blocked=[
                    dict(cloud=cloud, region=region)]))[0]]
                changed.add(k)
            if rnd < 3:
                ids = set()
                for sess, shard in zip(session._sessions,  # pylint: disable=protected-access
                                       session._batch.shards):  # pylint: disable=protected-access
                    if sess is not None and sess.last_dag_ids is not None:
                        ids.update(shard[d] for d in sess.last_dag_ids)
                if rnd > 0:
                    assert ids == prev_changed - session._fallback  # pylint: disable=protected-access
            prev_changed = changed


def run_all(devices=(0,), n_groups=1000):
    devices = list(devices)
    check_records(devices)
    check_mixed(devices, n_groups)
    check_ties(devices)
    check_most_regions(devices)
    check_session(devices)


def test_optimize_job_group_is_the_batch_path():
    """optimize_job_group copies no candidate table back for a group
    without an estimator, and equals the model."""
    runner.activate_catalog(scenarios.CATALOGS['multi6k'])
    calls = []
    real = engine.solve

    def spy(builder, device=0, want_tables=False):
        calls.append(want_tables)
        return real(builder, device=device, want_tables=want_tables)

    spec = scenarios.job_group_cases()[6]
    dag, tasks = _build(spec)
    engine.solve = spy
    try:
        sky.Optimizer.optimize_job_group(dag, quiet=True)
    finally:
        engine.solve = real
    assert calls == [False]
    assert _outcome(dag, tasks) == _model(spec)


def test_job_groups_one_and_two_shards():
    run_all([0])
    run_all([0, 0], n_groups=300)


@pytest.mark.parametrize('mode', [m for m in MODES if m != 'auto'])
def test_job_groups_in_every_kernel_mode(mode):
    stores = [runner.activate_catalog(spec) for spec in (
        reservation_scenarios.CATALOG, scenarios.CATALOGS['fuzzmany'])]
    stores.append(azmap_runner.activate())
    with runner.forced_paths(*stores, mode=mode):
        run_all([0], n_groups=200)


@pytest.mark.parametrize('path', ['8', '32'])
def test_job_groups_on_every_chain_path(path):
    """The chain DP's full evaluation; the chain on the block that places
    the last task (runner.CHAIN_PATHS)."""
    with runner.forced_paths(chain=path):
        run_all([0], n_groups=200)


# ---- SKYOPT_EINVAL -------------------------------------------------------------
def _group_problem():
    runner.activate_catalog(scenarios.CATALOGS['multi6k'])
    spec = scenarios.job_group_cases()[5]
    dag, _ = _build(spec)
    batch = opt_lib._Batch([dag], True, [0], [[]], job_groups=True)  # pylint: disable=protected-access
    return batch.builders[0]


def _optimize(b):
    packed = b.pack()
    sol = engine.Solution(packed, False)
    prob, csol = packed.c_problem(), sol.c_solution()
    lib = _native.load()
    return lib.skyopt_optimize_blocks(
        b.store.handle(0), ctypes.byref(prob), *packed.c_blocks(),
        ctypes.byref(csol), ctypes.byref(sol.stats))


def test_same_infra_einval():
    b = _group_problem()
    assert _optimize(b) == 0
    for kind in (-1, 3):
        b.dags[0]['is_chain'] = kind
        assert _optimize(b) == -1
        assert b'unknown kind' in _native.load().skyopt_last_error()
    b.dags[0]['is_chain'] = _native.DAG_SAME_INFRA
    b.add_task(b.tasks[0]['slot_begin'], b.tasks[0]['slot_end'], [0],
               [[0.0] * len(b.store.clouds)])
    b.dags[0]['task_end'] = len(b.tasks)
    assert _optimize(b) == -1
    assert b'has parents' in _native.load().skyopt_last_error()
    store = b.store
    with pytest.raises(_native.SkyoptError, match='needs regions'):
        engine.solve_tables(store, [[1.0], [2.0]], [[0], [0]], [[], []],
                            [[], []], [None, None], _native.DAG_SAME_INFRA,
                            True)
