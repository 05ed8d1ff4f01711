"""Placement contexts of a batch without a GPU: argument checks, each DAG's
slice of a mixed batch's packed problem against the problem stated alone
under the same process-wide state, the reservation block a slot names, the
bytes of a batch without contexts, the statement memo's key, and the entry
points that take the per-context reservation ranges."""
import contextlib
import copy
import ctypes

import numpy as np
import pytest

import skypilot_b200 as sky
from skypilot_b200 import _native
from skypilot_b200 import check
from skypilot_b200 import optimizer as opt_lib
from skypilot_b200 import placement_context
from skypilot_b200 import reservations
from skypilot_b200 import skypilot_config
from tests import reservation_scenarios
from tests import scenario_runner as runner

INV = reservation_scenarios.RESERVATION_INVENTORY
AWS_PRIO = {'aws': {'prioritize_reservations': True}}
BOTH_PRIO = {'aws': {'prioritize_reservations': True},
             'gcp': {'prioritize_reservations': True}}
PROXY = {'aws': {'ssh_proxy_command': {'us-east-2': 'ssh -W %h:%p a',
                                       'eu-west-1': 'ssh -W %h:%p b'}}}


@pytest.fixture(scope='module')
def store():
    return runner.activate_catalog(reservation_scenarios.CATALOG)


@contextlib.contextmanager
def process_state(ctx):
    """The process-wide state set to `ctx` (None fields keep theirs)."""
    saved = (check._enabled, skypilot_config._config,  # pylint: disable=protected-access
             reservations._records)  # pylint: disable=protected-access
    try:
        if ctx is not None and ctx.enabled_clouds is not None:
            check.set_enabled_clouds(list(ctx.enabled_clouds))
        if ctx is not None and ctx.config is not None:
            skypilot_config.set_config(ctx.config)
        if ctx is not None and ctx.reservations is not None:
            reservations.set_reservations(ctx.reservations)
        yield
    finally:
        check._enabled = saved[0]  # pylint: disable=protected-access
        skypilot_config.set_config(saved[1])
        reservations._records = saved[2]  # pylint: disable=protected-access


def _dags():
    """Single tasks, a chain with egress and a diamond; spot and on-demand,
    some pinned to a cloud."""
    specs = [
        dict(accelerators='V100', num_nodes=4),
        dict(accelerators='V100', num_nodes=4, use_spot=True),
        dict(cpus='8+', num_nodes=2),
        dict(infra='aws', accelerators='V100', num_nodes=6),
        dict(infra='gcp', accelerators='V100', num_nodes=3),
    ]
    dags = []
    for k, res in enumerate(specs):
        with sky.Dag() as dag:
            sky.Task(f's{k}', num_nodes=res.pop('num_nodes')).set_resources(
                sky.Resources(**res))
        dags.append(dag)
    for edges in ([(0, 1), (1, 2)], [(0, 1), (0, 2), (1, 3), (2, 3)]):
        n = max(max(e) for e in edges) + 1
        with sky.Dag() as dag:
            tasks = []
            for k in range(n):
                t = sky.Task(f'c{k}', num_nodes=1 + k % 3)
                t.set_resources(sky.Resources(
                    accelerators='V100' if k % 2 == 0 else None,
                    cpus=None if k % 2 == 0 else '8+'))
                t.set_outputs('s3://x', estimated_size_gigabytes=10 * (k + 1))
                tasks.append(t)
            for a, b in edges:
                tasks[a] >> tasks[b]  # pylint: disable=pointless-statement
        dags.append(dag)
    return dags


def _contexts():
    inv2 = copy.deepcopy(INV)
    for r in inv2:
        r['available'] += 3
    return [
        None,
        sky.PlacementContext(enabled_clouds=['aws'], config=AWS_PRIO,
                             reservations=INV),
        sky.PlacementContext(enabled_clouds=['aws', sky.GCP()],
                             config=BOTH_PRIO, reservations=inv2,
                             minimize=sky.OptimizeTarget.TIME),
        sky.PlacementContext(config=PROXY, reservations=[]),
        sky.PlacementContext(config=BOTH_PRIO, reservations=INV[:3]),
    ]


def test_argument_errors(store):
    del store
    dags = _dags()[:2]
    ctx = sky.PlacementContext()
    with pytest.raises(ValueError, match='2 DAGs'):
        sky.optimize_batch(dags, contexts=[ctx])
    with pytest.raises(ValueError, match='2 DAGs'):
        sky.Optimizer.batch_session(dags, contexts=[ctx, ctx, None])
    with pytest.raises(TypeError, match='PlacementContext'):
        sky.optimize_batch(dags, contexts=[ctx, {'config': {}}])
    # contexts go together with either kind of blocked list, which keep
    # their own checks
    with pytest.raises(ValueError, match='not both'):
        sky.optimize_batch(dags, blocked_resources=[],
                           blocked_resources_per_dag=[[], []],
                           contexts=[ctx, ctx])


def _alone(dag, ctx):
    """DAG stated alone under the process state set to `ctx`: its packed
    problem."""
    minimize_cost = not (ctx is not None and
                         ctx.minimize == sky.OptimizeTarget.TIME)
    with process_state(ctx):
        batch = opt_lib._Batch([dag], minimize_cost, [0], [[]])  # pylint: disable=protected-access
        return batch.builders[0].pack()


def _slice(packed, d):
    """DAG `d` of a packed problem: its slots, tasks and DAG record (slot
    and task indices relative to the DAG), its reservation block and the
    slots' flags."""
    dag = packed.dags[d].copy()
    t0, t1 = int(dag['task_begin']), int(dag['task_end'])
    tasks = packed.tasks[t0:t1].copy()
    s0, s1 = int(tasks['slot_begin'][0]), int(tasks['slot_end'][-1])
    slots = packed.slots[s0:s1].copy()
    tasks['slot_begin'] -= s0
    tasks['slot_end'] -= s0
    # parents and tariffs by content: their offsets are global
    n_clouds = len(packed.store.clouds)
    links = []
    for tk in tasks:
        pb, npar = int(tk['parent_begin']), int(tk['n_parents'])
        eb, sb = int(tk['edge_tariff_begin']), int(tk['src_tariff_begin'])
        links.append((packed.parents[pb:pb + npar].tobytes(),
                      packed.tariffs[eb:eb + npar * n_clouds].tobytes()
                      if npar else b'',
                      packed.tariffs[sb:sb + n_clouds].tobytes()
                      if sb >= 0 else b''))
    tasks['parent_begin'] = 0
    tasks['edge_tariff_begin'] = 0
    tasks['src_tariff_begin'] = np.minimum(tasks['src_tariff_begin'], 0)
    dag['task_begin'] -= t0
    dag['task_end'] -= t0
    pad = slots['pad_'].copy()
    flagged = sorted(set(int(p) for p in pad if p))
    assert len(flagged) <= 1
    if packed.reservation_ranges is None:
        block = packed.reservations[:packed.n_reservations]
    elif flagged:
        r = packed.reservation_ranges
        block = packed.reservations[r[flagged[0] - 1]:r[flagged[0]]]
    else:
        block = np.zeros(0, _native.RESERVATION_DTYPE)
    slots['pad_'] = 0
    # a slot's query ids are global: compare the queries themselves
    queries = [packed.queries[q].tobytes() if q >= 0 else None
               for q in slots['query']]
    slots['query'] = 0
    gates = [packed.queries[q].tobytes() if q >= 0 else None
             for q in slots['gate_query']]
    slots['gate_query'] = 0
    dag['blocked_begin'] = dag['blocked_end'] = 0
    return (slots.tobytes(), tasks.tobytes(), links, dag.tobytes(), queries,
            gates,
            (pad != 0).tolist(), block.tobytes() if flagged else b'')


@pytest.mark.parametrize('n_devices', [1, 2])
def test_mixed_batch_packs_each_dag_as_stated_alone(store, n_devices):
    del store
    dags = _dags()
    ctxs = _contexts()
    # every DAG under every context
    all_dags, all_ctxs = [], []
    for c in ctxs:
        for d in _dags():
            all_dags.append(d)
            all_ctxs.append(c)
    batch = opt_lib._Batch(all_dags, True, list(range(n_devices)),  # pylint: disable=protected-access
                           [[]] * len(all_dags), contexts=all_ctxs)
    # the AWS-only context cannot place the task pinned to GCP
    assert sorted(batch.errors) == [len(dags) + 4]
    n_flagged_blocks = set()
    for shard, b in zip(batch.shards, batch.builders):
        packed = b.pack()
        assert packed.reservation_ranges is not None
        r = packed.reservation_ranges
        assert (np.diff(r) >= 0).all() and r[-1] == packed.n_reservations
        for d, i in enumerate(shard):
            got = _slice(packed, d)
            want = _slice(_alone(all_dags[i], all_ctxs[i]), 0)
            assert got == want, (i, all_ctxs[i])
            n_flagged_blocks.update(
                int(p) for p in packed.slots['pad_'][:packed.n_slots] if p)
    # the reservation contexts with distinct inventories have blocks of
    # their own
    assert len(n_flagged_blocks) >= 2 * (n_devices == 1)
    del dags


def test_context_without_clouds_keeps_its_error(store):
    del store
    dags = _dags()[:3]
    ctxs = [None, sky.PlacementContext(enabled_clouds=[]),
            sky.PlacementContext(enabled_clouds=['gcp'])]
    dags[2].tasks[0].set_resources(sky.Resources(infra='aws', cpus='2+'))
    batch = opt_lib._Batch(dags, True, [0], [[]] * 3, contexts=ctxs)  # pylint: disable=protected-access
    assert sorted(batch.errors) == [1, 2]
    for i, ctx in ((1, ctxs[1]), (2, ctxs[2])):
        with process_state(ctx):
            with pytest.raises(type(batch.errors[i])) as info:
                sky.Optimizer.optimize(dags[i], quiet=True)
        assert str(info.value) == str(batch.errors[i])
    assert isinstance(batch.errors[1], sky.exceptions.NoCloudAccessError)
    assert batch.shards == [[0]]
    assert len(batch.builders[0].dags) == 1


def test_batch_without_contexts_packs_the_same_bytes(store):
    """No contexts: the problem of the process-wide state, stated and
    packed as before (one table read when packing, no ranges). Contexts that
    all defer to the process: the same bytes plus one range over the
    table."""
    del store
    skypilot_config.set_config(BOTH_PRIO)
    reservations.set_reservations(INV)
    try:
        plain = opt_lib._Batch(_dags(), True, [0], [[]] * 7)  # pylint: disable=protected-access
        deferring = opt_lib._Batch(_dags(), True, [0], [[]] * 7,  # pylint: disable=protected-access
                                   contexts=[None] * 7)
        p, q = plain.builders[0].pack(), deferring.builders[0].pack()
    finally:
        reservations.set_reservations(None)
        skypilot_config.set_config(None)
    assert p.reservation_ranges is None
    assert p.c_blocks() == (None, 0)
    assert q.c_blocks()[1] == 1
    assert p.n_reservations > 0 and p.slots['pad_'].any()
    for name in ('queries', 'acc_sets', 'slots', 'tasks', 'parents',
                 'tariffs', 'blocked', 'dags', 'reservations'):
        assert getattr(p, name).tobytes() == getattr(q, name).tobytes(), name
    assert list(q.reservation_ranges) == [0, p.n_reservations]


def test_memo_keys_follow_config_content(store):
    del store
    a = sky.PlacementContext(config=copy.deepcopy(AWS_PRIO))
    a2 = sky.PlacementContext(config=copy.deepcopy(AWS_PRIO))
    b = sky.PlacementContext(config=BOTH_PRIO)
    empty = sky.PlacementContext(config={})
    keys = {}
    for name, ctx in (('a', a), ('a2', a2), ('b', b), ('empty', empty),
                      ('none', None)):
        with placement_context.active(ctx):
            keys[name] = skypilot_config.key()
    assert keys['a'] == keys['a2']
    assert len({keys['a'], keys['b'], keys['empty'], keys['none']}) == 4
    assert keys['none'] == skypilot_config.generation()
    # a task's recorded statement is replayed under an equal config and
    # stated again under another one
    dag = _dags()[0]
    task = dag.tasks[0]
    seen = []
    for ctx in (a, a2, b):
        opt_lib._Batch([dag], True, [0], [[]], contexts=[ctx])  # pylint: disable=protected-access
        seen.append(task.__dict__['_stated'])
    assert seen[0] is seen[1]
    assert seen[2] is not seen[1] and seen[2][1] != seen[1][1]
    # the active context does not reach another thread
    with placement_context.active(b):
        got = opt_lib._run_shards([skypilot_config.key])  # pylint: disable=protected-access
    assert got == [skypilot_config.generation()]


def test_contexts_are_read_by_the_process_readers(store):
    del store
    ctx = sky.PlacementContext(enabled_clouds=['gcp', 'aws'],
                               config=AWS_PRIO, reservations=INV[:1])
    with placement_context.active(ctx):
        names = [str(c).lower() for c in
                 check.get_cached_enabled_clouds_or_refresh()]
        assert names == ['gcp', 'aws']
        assert reservations.need_to_query()
        assert reservations.records() == (reservations.as_record(INV[0]),)
        assert skypilot_config.get_nested(('aws', 'prioritize_reservations'))
    assert not reservations.need_to_query()
    with placement_context.active(sky.PlacementContext(enabled_clouds=[])):
        with pytest.raises(sky.exceptions.NoCloudAccessError):
            check.get_cached_enabled_clouds_or_refresh(
                raise_if_no_cloud_access=True)


def test_reservation_blocks_entry_points():
    """Per-context blocks travel as arguments of two added functions; the
    records and SkyoptProblem keep their layout and the ABI version."""
    assert _native.ABI_VERSION == 4
    assert _native.SLOT_DTYPE.itemsize == 80
    assert _native.SLOT_DTYPE.fields['pad_'][1] == 52
    assert _native.RESERVATION_DTYPE.itemsize == 16
    names = [n for n, _ in _native.Problem._fields_]  # pylint: disable=protected-access
    assert names[-2:] == ['reservations', 'n_reservations']
    assert ctypes.sizeof(_native.Problem) == 144
    lib = _native.load()
    assert lib.skyopt_abi_version() == 4
    for name in ('skyopt_optimize_blocks', 'skyopt_session_open_blocks'):
        assert name in _native.EXPORTS
        argtypes = getattr(lib, name).argtypes
        # (catalog, problem, ranges, n_ranges, solution, stats[, out])
        assert argtypes[2] is ctypes.c_void_p and argtypes[3] is ctypes.c_int
        assert argtypes[1]._type_ is _native.Problem  # pylint: disable=protected-access
        assert argtypes[4]._type_ is _native.Solution  # pylint: disable=protected-access
