"""New reservation inventories for an open batch session, on the device:
rounds that change inventories (counts, dropped records, added zones and
clouds, a targeted reservation named and unnamed) together with blocked
lists, against one Optimizer.optimize per DAG under its context at that
moment, with exactly the forced DAGs and the DAGs whose candidate values
change re-solved -- in every kernel mode, on every chain-DP path, on one
shard and on two -- plus changes that must
re-solve nothing, context changes that state everything again, and the
argument checks of skyopt_session_update_dags."""
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
from tests.test_gpu_batch_contexts import _single

pytestmark = pytest.mark.gpu
MODES = ['auto', 'fast-split', 'fast-noprune', 'queue', 'tile']
INV = reservation_scenarios.RESERVATION_INVENTORY
AWS_PRIO = {'aws': {'prioritize_reservations': True}}
BOTH_PRIO = {'aws': {'prioritize_reservations': True},
             'gcp': {'prioritize_reservations': True}}
SPECIFIC = {'aws': {'specific_reservations': ['cr-tgt-w2c']},
            'gcp': {'prioritize_reservations': True}}
# records a round may add: other zones of the fixture's types, and clouds
EXTRA = [
    dict(cloud='aws', instance_type='p3.2xlarge', zone='us-west-2a',
         name='cr-new-w2a', available=2),
    dict(cloud='aws', instance_type='p3.2xlarge', zone='us-east-1a',
         name='cr-new-e1a', available=5),
    dict(cloud='aws', instance_type='m6i.2xlarge', zone='us-east-2a',
         name='cr-cpu-e2a', available=3),
    dict(cloud='gcp', instance_type='n1-highmem-8', zone='us-central1-a',
         name='projects/p/reservations/g-c1a', available=2),
]


def _kinds():
    """The fixed part of each shared context: (enabled clouds, config,
    objective); its inventory changes round by round."""
    t = sky.OptimizeTarget
    return [
        (('aws', 'gcp'), BOTH_PRIO, None),
        (('aws',), AWS_PRIO, None),
        (('aws', 'gcp', 'azure'), SPECIFIC, None),
        (('aws', 'gcp'), BOTH_PRIO, t.TIME),
        # a config that enables no reservation: no inventory counts
        (('aws', 'gcp'), {}, None),
    ]


def _mutate(inventory, rng, rnd):
    """One round's change of an inventory: counts, dropped records, added
    zones and clouds, the targeted AWS reservation renamed in or out of
    specific_reservations."""
    out = [dict(r) for r in inventory]
    kind = rnd % 4
    if kind == 0:
        for r in out:
            if rng.uniform() < 0.5:
                r['available'] = int(rng.integers(0, 9))
    elif kind == 1 and out:
        keep = rng.uniform(size=len(out)) < 0.6
        out = [r for r, k in zip(out, keep) if k]
    elif kind == 2:
        out += [dict(r) for r in EXTRA if rng.uniform() < 0.7 and
                all(q['name'] != r['name'] for q in out)]
    for r in out:
        if r['name'] in ('cr-tgt-w2c', 'cr-tgt-out') and kind == 3:
            r['name'] = ('cr-tgt-out' if r['name'] == 'cr-tgt-w2c' else
                         'cr-tgt-w2c')
    return out


def _contexts(kinds, inventories):
    return [sky.PlacementContext(enabled_clouds=list(c), config=cfg,
                                 reservations=inv, minimize=m)
            for (c, cfg, m), inv in zip(kinds, inventories)]


def _values(specs, contexts, devices):
    """Every DAG's unblocked candidate values (bytes per task) from a fresh
    solve with tables, or None off the device."""
    dags = [runner.build_dag(s)[0] for s in specs]
    batch = opt_lib._Batch(dags, True, devices, [[]] * len(dags),  # pylint: disable=protected-access
                           contexts=contexts)
    out = [None] * len(dags)
    for k, b in enumerate(batch.builders):
        if not b.dags or b.n_slots == 0:
            continue
        sol = engine.solve(b, device=devices[k], want_tables=True)
        for i in batch.shards[k]:
            first = batch.first_task[i]
            out[i] = tuple(sol.task_table(first + j)['value'].tobytes()
                           for j in range(len(dags[i].tasks)))
    return out


def _fixture_specs():
    """The reservation fixture's scenarios that the reference constructs
    (a few are refused with ValueError while the request is built)."""
    out = []
    for s in reservation_runner.optimizer_scenarios():
        try:
            runner.build_dag(s)
        except ValueError:
            continue
        out.append(s)
    return out


def _specs(n=300):
    resv = _fixture_specs()
    by_name = {s['name']: s for s in scenarios.basic_scenarios()}
    shaped = [by_name[m] for m in ('cfg2_chain8', 'chain3_mixed',
                                   'cfg3_diamond', 'ordered_list')]
    specs = failover._cfg5_specs(n, seed=17)  # pylint: disable=protected-access
    for k, s in enumerate(shaped):
        specs.insert(41 * k + 3, dict(s, name=f'shaped_{k}'))
    return resv + specs


def check_rounds(devices):
    runner.activate_catalog(reservation_scenarios.CATALOG)
    specs = _specs()
    n_fixture = len(_fixture_specs())
    kinds = _kinds()
    # the fixture scenarios keep their own config under a context each
    own = [(('aws', 'gcp', 'azure'), s.get('config') or {},
            sky.OptimizeTarget.TIME if s.get('minimize') == 'time' else None)
           for s in specs[:n_fixture]]
    all_kinds = own + kinds
    kind_of = list(range(n_fixture)) + [
        n_fixture + k % len(kinds) for k in range(len(specs) - n_fixture)]
    inventories = ([s.get('reservations') or [] for s in specs[:n_fixture]] +
                   [copy.deepcopy(INV) for _ in kinds])
    ordered = {k for k, s in enumerate(specs)
               if s['name'].startswith('shaped_3')}
    built = [runner.build_dag(s) for s in specs]
    rng = np.random.default_rng(41)
    wild = [list(s.get('blocked', [])) for s in specs]
    forced = set()
    ctxs = _contexts(all_kinds, inventories)
    contexts = [ctxs[kind_of[i]] for i in range(len(specs))]
    values = _values(specs, contexts, devices)
    n_repriced = 0
    with sky.Optimizer.batch_session([d for d, _ in built], devices=devices,
                                     contexts=contexts) as bs:
        for rnd in range(6):
            lists = [runner.blocked_list({'blocked': w}) or [] for w in wild]
            if rnd:
                # two shared contexts and two fixture ones change
                picks = list(n_fixture + rng.choice(len(kinds), size=2,
                                                    replace=False))
                picks += list(rng.choice(n_fixture, size=2, replace=False))
                for k in picks:
                    inventories[k] = _mutate(inventories[k], rng, rnd)
                ctxs = _contexts(all_kinds, inventories)
                contexts = [ctxs[kind_of[i]] for i in range(len(specs))]
                new_values = _values(specs, contexts, devices)
                model = {i for i in range(len(specs))
                         if new_values[i] != values[i]}
                values = new_values
                before = list(bs._sessions)  # pylint: disable=protected-access
            out = bs.optimize(lists, return_exceptions=True,
                              contexts=contexts)
            if rnd:
                assert all(a is b for a, b in zip(before, bs._sessions))  # pylint: disable=protected-access
                on_device = {i for shard in bs._batch.shards for i in shard}  # pylint: disable=protected-access
                want = ((forced | model) & on_device) - ordered
                assert failover._device_ids(bs) == want, (  # pylint: disable=protected-access
                    rnd, sorted(failover._device_ids(bs) ^ want)[:8])  # pylint: disable=protected-access
                n_repriced += len(model - forced)
            for k, (o, (_, tasks)) in enumerate(zip(out, built)):
                assert failover._outcome(o, tasks) == _single(  # pylint: disable=protected-access
                    specs[k], contexts[k], lists[k]), (rnd, specs[k]['name'])
            live = [k for k, o in enumerate(out)
                    if not isinstance(o, Exception)]
            forced = set()
            for k in rng.choice(live, size=max(1, len(live) // 10),
                                replace=False):
                k = int(k)
                tasks = built[k][1]
                rec = runner.res_record(
                    tasks[int(rng.integers(len(tasks)))].best_resources)
                wild[k].append(failover._wildcard(  # pylint: disable=protected-access
                    rec, failover._WILD_KINDS[(rnd + k) % 4]))  # pylint: disable=protected-access
                forced.add(k)
    assert n_repriced >= 10


def _one_task(num_nodes=4, zero_time=False, **res):
    with sky.Dag() as dag:
        t = sky.Task('t', num_nodes=num_nodes)
        t.set_resources(sky.Resources(**res))
        if zero_time:
            t.set_time_estimator(lambda _: 0.0)
    return dag, [t]


def check_quiet_changes(devices):
    """Inventory changes that change no candidate value re-solve nothing."""
    runner.activate_catalog(reservation_scenarios.CATALOG)
    rec = dict(cloud='aws', instance_type='p3.2xlarge', zone='us-west-2b',
               name='cr-q', available=10)
    t = sky.OptimizeTarget

    def ctx(config, count, minimize=None):
        return sky.PlacementContext(
            enabled_clouds=['aws'], config=config, minimize=minimize,
            reservations=[dict(rec, available=count)])

    cases = [
        # TIME: reserved nodes never enter the objective
        (dict(infra='aws', instance_type='p3.2xlarge'), False,
         lambda c: ctx(AWS_PRIO, c, t.TIME), (10, 0)),
        # a config that enables no reservation
        (dict(infra='aws', instance_type='p3.2xlarge'), False,
         lambda c: ctx({}, c), (10, 2)),
        # max(4 - r, 0) stays 0
        (dict(infra='aws', instance_type='p3.2xlarge'), False,
         lambda c: ctx(AWS_PRIO, c), (10, 12)),
        # a zero-cost candidate (no runtime) stays zero
        (dict(infra='aws', instance_type='p3.2xlarge'), True,
         lambda c: ctx(AWS_PRIO, c), (10, 1)),
    ]
    for res, zero, make, (a, b) in cases:
        built = [_one_task(zero_time=zero, **res) for _ in range(3)]
        dags = [d for d, _ in built]
        first = [make(a)] * 3
        with sky.Optimizer.batch_session(dags, devices=devices,
                                         contexts=first) as bs:
            bs.optimize(return_exceptions=True)
            sessions = list(bs._sessions)  # pylint: disable=protected-access
            second = [make(b)] * 3
            out = bs.optimize(return_exceptions=True, contexts=second)
            assert all(x is y for x, y in zip(sessions, bs._sessions))  # pylint: disable=protected-access
            assert failover._device_ids(bs) == set(), (res, zero, a, b)  # pylint: disable=protected-access
            for o, (_, tasks) in zip(out, built):
                assert failover._outcome(o, tasks) == _outcome_alone(  # pylint: disable=protected-access
                    res, zero, second[0])
    # and a count that matters re-solves exactly its DAGs
    built = [_one_task(**dict(infra='aws', instance_type='p3.2xlarge'))
             for _ in range(4)]
    with sky.Optimizer.batch_session([d for d, _ in built], devices=devices,
                                     contexts=[ctx(AWS_PRIO, 0)] * 4) as bs:
        bs.optimize()
        new = [ctx(AWS_PRIO, 0), ctx(AWS_PRIO, 2), ctx(AWS_PRIO, 0),
               ctx(AWS_PRIO, 3)]
        out = bs.optimize(contexts=new)
        assert failover._device_ids(bs) == {1, 3}  # pylint: disable=protected-access
        for o, (_, tasks), c in zip(out, built, new):
            assert failover._outcome(o, tasks) == _outcome_alone(  # pylint: disable=protected-access
                dict(infra='aws', instance_type='p3.2xlarge'), False, c)


def _outcome_alone(res, zero, ctx):
    from tests.test_batch_contexts import process_state  # pylint: disable=import-outside-toplevel
    dag, tasks = _one_task(zero_time=zero, **res)
    target = ctx.minimize or sky.OptimizeTarget.COST
    with process_state(ctx):
        sky.Optimizer.optimize(dag, target, quiet=True)
    return failover._outcome(dag, tasks)  # pylint: disable=protected-access


def check_full_solves(devices):
    """A changed config, set of clouds or objective states everything
    again under the new contexts."""
    runner.activate_catalog(reservation_scenarios.CATALOG)
    specs = [s for s in reservation_runner.optimizer_scenarios()
             if s['name'] in ('aws_prio_v100_n4', 'chain3_egress',
                              'diamond4', 'gcp_prio_v100_n3')]
    base = sky.PlacementContext(enabled_clouds=['aws', 'gcp'],
                                config=BOTH_PRIO, reservations=INV)
    changes = [
        sky.PlacementContext(enabled_clouds=['aws', 'gcp'], config=AWS_PRIO,
                             reservations=INV),
        sky.PlacementContext(enabled_clouds=['aws'], config=BOTH_PRIO,
                             reservations=INV),
        sky.PlacementContext(enabled_clouds=['aws', 'gcp'], config=BOTH_PRIO,
                             reservations=INV,
                             minimize=sky.OptimizeTarget.TIME),
    ]
    built = [runner.build_dag(s) for s in specs]
    for change in changes:
        with sky.Optimizer.batch_session([d for d, _ in built],
                                         devices=devices,
                                         contexts=[base] * len(specs)) as bs:
            bs.optimize(return_exceptions=True)
            before = list(bs._sessions)  # pylint: disable=protected-access
            contexts = [base] * (len(specs) - 1) + [change]
            out = bs.optimize(return_exceptions=True, contexts=contexts)
            assert not any(a is b for a, b in zip(before, bs._sessions)  # pylint: disable=protected-access
                           if a is not None)
            for k, (o, (_, tasks)) in enumerate(zip(out, built)):
                assert failover._outcome(o, tasks) == _single(  # pylint: disable=protected-access
                    specs[k], contexts[k])


def run_all(devices=(0,)):
    devices = list(devices)
    check_rounds(devices)
    check_quiet_changes(devices)
    check_full_solves(devices)


@pytest.mark.parametrize('mode', MODES)
def test_reservation_updates_in_every_kernel_mode(mode):
    store = runner.activate_catalog(reservation_scenarios.CATALOG)
    with runner.forced_paths(store, mode=mode):
        run_all([0])
        run_all([0, 0])


@pytest.mark.parametrize('path', ['8', '32'])
def test_reservation_updates_on_every_chain_path(path):
    """The chain DP's full evaluation; the chain on the block that places
    the last task (runner.CHAIN_PATHS)."""
    with runner.forced_paths(chain=path):
        run_all([0])


# ---- skyopt_session_update_dags argument checks -----------------------------
def test_update_dags_rejects_bad_arguments():
    runner.activate_catalog(reservation_scenarios.CATALOG)
    dags = [_one_task(num_nodes=4, infra='aws', instance_type='p3.2xlarge')[0]
            for _ in range(3)]
    ctx = sky.PlacementContext(enabled_clouds=['aws', 'gcp'],
                               config=BOTH_PRIO, reservations=INV)
    batch = opt_lib._Batch(dags, True, [0], [[]] * 3, contexts=[ctx] * 3)  # pylint: disable=protected-access
    session = engine.Session(batch.builders[0])
    try:
        lib = _native.load()
        packed = session.packed
        first = session.solution
        assert packed.n_reservations >= 2 and packed.slots['pad_'].any()
        blocked = np.zeros(2, dtype=_native.BLOCKED_DTYPE)
        blocked[:] = -1

        def call(resv=None, rr=None, pad=None, n_slots=None, forced=(),
                 ranges=None):
            resv = packed.reservations.copy() if resv is None else resv
            rr = packed.reservation_ranges.copy() if rr is None else rr
            pad = (np.ascontiguousarray(packed.slots['pad_'][:packed.n_slots])
                   if pad is None else pad)
            ranges = np.zeros(2 * 3, np.int32) if ranges is None else ranges
            ids = np.asarray(list(forced) or [0], dtype=np.int32)
            out_ids = np.zeros(3, np.int32)
            out_n = np.zeros(1, np.int32)
            sol = engine.Solution(packed, False)
            csol = sol.c_solution()
            return lib.skyopt_session_update_dags(
                session._handle, blocked.ctypes.data, 2,  # pylint: disable=protected-access
                np.ascontiguousarray(ranges, np.int32).ctypes.data,
                ids.ctypes.data, len(forced), resv.ctypes.data, len(resv),
                rr.ctypes.data, len(rr) - 1,
                np.ascontiguousarray(pad, np.int32).ctypes.data,
                packed.n_slots if n_slots is None else n_slots,
                out_ids.ctypes.data, out_n.ctypes.data, ctypes.byref(csol),
                ctypes.byref(sol.stats))

        unsorted = packed.reservations.copy()
        unsorted[[0, 1]] = unsorted[[1, 0]]
        repeated = packed.reservations.copy()
        repeated[1] = repeated[0]
        bad_key = packed.reservations.copy()
        bad_key['inst_id'][0] = -1
        pad = np.ascontiguousarray(packed.slots['pad_'][:packed.n_slots])
        cases = {
            'descending': dict(rr=np.array([2, 0], np.int32)),
            'outside': dict(rr=np.array([0, len(packed.reservations) + 1],
                                        np.int32)),
            'unsorted': dict(resv=unsorted),
            'repeated': dict(resv=repeated),
            'bad_key': dict(resv=bad_key),
            'pad_high': dict(pad=np.where(pad > 0, 2, 0)),
            'pad_negative': dict(pad=np.where(pad > 0, -1, 0)),
            'n_slots': dict(n_slots=packed.n_slots - 1),
            'forced_out': dict(forced=[3]),
            'forced_negative': dict(forced=[-1]),
            'forced_twice': dict(forced=[1, 1]),
            'range_outside': dict(ranges=np.array([0, 3, 0, 0, 0, 0])),
            'range_negative': dict(ranges=np.array([0, 0, -1, 0, 0, 0])),
            'range_reversed': dict(ranges=np.array([0, 0, 0, 0, 2, 1])),
        }
        for name, kw in cases.items():
            assert call(**kw) == -1, name  # SKYOPT_EINVAL
            assert lib.skyopt_last_error()
        # nothing was launched or replaced: the same inventory re-prices
        # nothing and the first plan comes back without a gather or solve
        sol = session.update_dags([], [(0, 0)] * 3, [])
        assert session.last_dag_ids == []
        assert sol.stats.total_launches == 1  # the re-price pass only
        assert (sol.dag['objective'] == first.dag['objective']).all()
        assert (sol.chosen_index[:packed.n_tasks] ==
                first.chosen_index[:packed.n_tasks]).all()
    finally:
        session.close()
