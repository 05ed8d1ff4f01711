"""New reservation inventories for an open batch session, without a GPU:
argument checks of `BatchOptimizerSession.optimize(contexts=...)`, the
reservation table, blocks and slot flags an update hands the device against
what a fresh open under the new contexts packs, which context changes
re-price and which state everything again, and the added entry point."""
import copy
import ctypes

import numpy as np
import pytest

import skypilot_b200 as sky
from skypilot_b200 import _native
from skypilot_b200 import optimizer as opt_lib
from tests import reservation_scenarios
from tests import scenario_runner as runner
from tests.test_batch_contexts import _dags

INV = reservation_scenarios.RESERVATION_INVENTORY
AWS_INV = [r for r in INV if r['cloud'] == 'aws']
GCP_INV = [r for r in INV if r['cloud'] == 'gcp']
BOTH_PRIO = {'aws': {'prioritize_reservations': True},
             'gcp': {'prioritize_reservations': True}}
SPECIFIC = {'aws': {'specific_reservations': ['cr-tgt-w2c']},
            'gcp': {'prioritize_reservations': True}}


@pytest.fixture(scope='module')
def store():
    return runner.activate_catalog(reservation_scenarios.CATALOG)


def _ctx(config, inventory, clouds=('aws', 'gcp'), minimize=None):
    return sky.PlacementContext(enabled_clouds=list(clouds),
                                config=copy.deepcopy(config),
                                reservations=inventory, minimize=minimize)


def _renamed(inventory, old, new):
    return [dict(r, name=new) if r['name'] == old else r for r in inventory]


def test_argument_errors(store):
    del store
    dags = _dags()[:2]
    session = sky.Optimizer.batch_session(dags)
    with pytest.raises(ValueError, match='2 DAGs'):
        session.optimize(contexts=[sky.PlacementContext()])
    with pytest.raises(ValueError, match='2 DAGs'):
        session.optimize(contexts=[None, None, None])
    with pytest.raises(TypeError, match='PlacementContext'):
        session.optimize(contexts=[None, {'reservations': []}])
    # nothing was opened by the refused calls
    assert session._batch is None  # pylint: disable=protected-access


def _base_contexts():
    return [
        _ctx(BOTH_PRIO, AWS_INV),
        _ctx(SPECIFIC, INV),
        _ctx(BOTH_PRIO, INV[:3]),
        None,
    ]


def _cases():
    """name -> (old contexts, new contexts) that differ in reservation
    inventories only."""
    base = _base_contexts()

    def with_inventory(k, inventory, ctxs=None):
        out = list(ctxs or base)
        c = out[k]
        out[k] = sky.PlacementContext(
            enabled_clouds=c.enabled_clouds, config=c.config,
            reservations=inventory, minimize=c.minimize)
        return out

    renamed = with_inventory(1, _renamed(INV, 'cr-tgt-w2c', 'cr-tgt-other'))
    return {
        # an AWS-only inventory gains GCP records: GCP slots get flags
        'add_cloud': (base, with_inventory(0, AWS_INV + GCP_INV)),
        'remove_all': (base, with_inventory(1, [])),
        # the targeted reservation leaves specific_reservations, and comes
        # back
        'rename_out': (base, renamed),
        'rename_in': (renamed, base),
        # the first context takes the third's inventory: the blocks merge
        # and every later block moves down
        'renumber': (base, with_inventory(0, INV[:3])),
        'counts': (base, with_inventory(
            2, [dict(r, available=r['available'] + 1) for r in INV[:3]])),
        # a DAG that deferred to the process takes an inventory of its own
        'own_inventory': (base, base[:3] + [
            sky.PlacementContext(reservations=INV[:1])]),
    }


def _per_dag(ctxs, n):
    return [ctxs[k % len(ctxs)] for k in range(n)]


@pytest.mark.parametrize('n_devices', [1, 2])
@pytest.mark.parametrize('name', sorted(_cases()))
def test_update_packs_what_a_fresh_open_packs(store, name, n_devices):
    """After restating an open batch's reservation blocks under new contexts
    and repacking, the shard's reservation table, its ranges and every
    slot's flag are byte-equal to a fresh batch's under those contexts; the
    rest of the problem is untouched."""
    del store
    old_ctxs, new = _cases()[name]
    dags = _dags() + _dags()
    devices = list(range(n_devices))
    lists = [[]] * len(dags)
    old = opt_lib._Batch(dags, True, devices, lists,  # pylint: disable=protected-access
                         contexts=_per_dag(old_ctxs, len(dags)))
    packed = [b.pack() for b in old.builders]
    before = [p.slots.copy() for p in packed]
    old.restate_reservations(_per_dag(new, len(dags)))
    fresh = opt_lib._Batch(_dags() + _dags(), True, devices, lists,  # pylint: disable=protected-access
                           contexts=_per_dag(new, len(dags)))
    changed = False
    for k, (b, p) in enumerate(zip(old.builders, packed)):
        p.repack_reservations(b)
        want = fresh.builders[k].pack()
        assert old.shards[k] == fresh.shards[k]
        assert p.n_reservations == want.n_reservations
        assert p.reservations.tobytes() == want.reservations.tobytes()
        assert (p.reservation_ranges.tobytes() ==
                want.reservation_ranges.tobytes())
        assert p.slots.tobytes() == want.slots.tobytes()
        for field in ('queries', 'tasks', 'dags', 'blocked'):
            assert (getattr(p, field).tobytes() ==
                    getattr(want, field).tobytes()), field
        # only the flags can differ from the first pack
        for f in _native.SLOT_DTYPE.names:
            if f != 'pad_':
                assert p.slots[f].tobytes() == before[k][f].tobytes(), f
        changed |= not np.array_equal(p.slots['pad_'], before[k]['pad_'])
    if name in ('add_cloud', 'remove_all', 'renumber'):
        assert changed, name


def test_gcp_slots_take_flags_when_gcp_records_arrive(store):
    del store
    dags = _dags()
    old = opt_lib._Batch(dags, True, [0], [[]] * len(dags),  # pylint: disable=protected-access
                         contexts=[_ctx(BOTH_PRIO, AWS_INV)] * len(dags))
    b = old.builders[0]
    p = b.pack()
    gcp = store_cloud_index('gcp')
    gcp_slots = p.slots['cloud'][:p.n_slots] == gcp
    assert gcp_slots.any() and not p.slots['pad_'][:p.n_slots][gcp_slots].any()
    old.restate_reservations([_ctx(BOTH_PRIO, AWS_INV + GCP_INV)] *
                             len(dags))
    p.repack_reservations(b)
    on_demand = p.slots['use_spot'][:p.n_slots] == 0
    assert (p.slots['pad_'][:p.n_slots][gcp_slots & on_demand] == 1).all()


def store_cloud_index(name):
    return sky.catalog.get_store().cloud(name).index


def test_statement_keys_classify_context_changes():
    t = sky.OptimizeTarget
    a = _ctx(BOTH_PRIO, INV)
    same = [
        _ctx(BOTH_PRIO, INV[:2]),
        _ctx(copy.deepcopy(BOTH_PRIO), []),
        _ctx(BOTH_PRIO, None),
    ]
    for b in same:
        assert opt_lib._same_statements([a], [b])  # pylint: disable=protected-access
    differ = [
        _ctx(SPECIFIC, INV),
        _ctx(BOTH_PRIO, INV, clouds=('aws',)),
        _ctx(BOTH_PRIO, INV, clouds=('gcp', 'aws')),
        _ctx(BOTH_PRIO, INV, minimize=t.TIME),
        sky.PlacementContext(reservations=INV),
    ]
    for b in differ:
        assert not opt_lib._same_statements([a], [b])  # pylint: disable=protected-access
    # None stands for a context that defers every field to the process
    assert opt_lib._same_statements(  # pylint: disable=protected-access
        [None], [sky.PlacementContext(reservations=INV)])
    assert opt_lib._same_statements(  # pylint: disable=protected-access
        [sky.PlacementContext(reservations=[])], [None])
    assert not opt_lib._same_statements(  # pylint: disable=protected-access
        [None], [sky.PlacementContext(minimize=t.TIME)])
    # a session opened without contexts states everything again
    assert not opt_lib._same_statements(None, [None])  # pylint: disable=protected-access


def test_update_entry_point():
    """skyopt_session_update_dags: bound, exported, ABI and layouts kept."""
    assert _native.ABI_VERSION == 4
    assert _native.SLOT_DTYPE.itemsize == 80
    assert _native.RESERVATION_DTYPE.itemsize == 16
    assert 'skyopt_session_update_dags' in _native.EXPORTS
    lib = _native.load()
    assert lib.skyopt_abi_version() == 4
    p, i = ctypes.c_void_p, ctypes.c_int
    argtypes = lib.skyopt_session_update_dags.argtypes
    # (session, blocked, n_blocked, ranges, forced_ids, n_forced,
    #  reservations, n_reservations, reservation_ranges, n_blocks,
    #  slot_pad, n_slots, out_ids, out_n_ids, solution, stats)
    assert argtypes[:14] == [p, p, i, p, p, i, p, i, p, i, p, i, p, p]
    assert argtypes[14]._type_ is _native.Solution  # pylint: disable=protected-access
    assert argtypes[15]._type_ is _native.Stats  # pylint: disable=protected-access
