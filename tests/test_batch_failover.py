"""Per-DAG blocked lists of a batch without a GPU: argument checks of
optimize_batch and the batch session, each DAG's own blocked range in the
stated problem, change detection on packed entries, and the C ABI of
skyopt_session_resolve_dags."""
import ctypes

import pytest

import skypilot_b200 as sky
from skypilot_b200 import _native
from skypilot_b200 import optimizer as opt_lib
from skypilot_b200.utils import registry
from tests import scenario_runner as runner
from tests import scenarios


@pytest.fixture(scope='module')
def store():
    return runner.activate_catalog(scenarios.CATALOGS['multi6k'])


def _dags(n):
    dags = []
    for k in range(n):
        with sky.Dag() as dag:
            sky.Task(f't{k}').set_resources(
                sky.Resources(accelerators=['V100', 'T4', 'A100'][k % 3]))
        dags.append(dag)
    return dags


def _blocked(**kw):
    if 'cloud' in kw:
        kw['cloud'] = registry.CLOUD_REGISTRY.from_str(kw['cloud'])
    r = sky.Resources(**kw)
    r._use_spot_specified = False  # pylint: disable=protected-access
    return r


def test_per_dag_lists_exclude_the_shared_list(store):
    del store
    dags = _dags(2)
    with pytest.raises(ValueError, match='not both'):
        sky.optimize_batch(dags, blocked_resources=[],
                           blocked_resources_per_dag=[[], []])
    with pytest.raises(ValueError, match='2 DAGs'):
        sky.optimize_batch(dags, blocked_resources_per_dag=[[]])
    with pytest.raises(ValueError, match='2 DAGs'):
        sky.Optimizer.batch_session(dags).optimize([[], [], []])


@pytest.mark.parametrize('n_devices', [1, 2])
def test_each_dag_states_its_own_blocked_range(store, n_devices):
    """Mixed lists (empty ones, a cloud-less wildcard that expands to one
    entry per cloud, one Resources object shared by several lists): every
    DAG's range in its shard holds exactly the entries of its own list."""
    aws_region = _blocked(cloud='aws', region='us-east-1')
    shared = _blocked(accelerators='V100')
    any_region = _blocked(region='us-east-1')
    lists = [[], [aws_region], [shared], [], [shared, any_region],
             [aws_region, shared], []]
    dags = _dags(len(lists))
    batch = opt_lib._Batch(dags, True, list(range(n_devices)), lists)  # pylint: disable=protected-access
    assert len(opt_lib._packed_blocked(store, [any_region])) == len(  # pylint: disable=protected-access
        store.clouds)
    for shard, b in zip(batch.shards, batch.builders):
        assert len(b.dags) == len(shard)
        end = 0
        for d, i in enumerate(shard):
            dag = b.dags[d]
            assert dag['blocked_begin'] == end
            end = dag['blocked_end']
            got = b.blocked[dag['blocked_begin']:dag['blocked_end']]
            assert got == opt_lib._packed_blocked(store, lists[i])  # pylint: disable=protected-access
        assert end == len(b.blocked)
        packed = b.pack()
        assert list(packed.dags['blocked_begin'][:len(shard)]) == [
            b.dags[d]['blocked_begin'] for d in range(len(shard))]
        assert list(packed.dags['blocked_end'][:len(shard)]) == [
            b.dags[d]['blocked_end'] for d in range(len(shard))]
    assert sorted(i for shard in batch.shards for i in shard) == list(
        range(len(lists)))


def test_one_shared_list_is_stated_for_every_dag(store):
    """Without per-DAG lists every DAG takes the one list, as before."""
    blocked = [_blocked(cloud='aws', region='us-east-1'),
               _blocked(accelerators='T4')]
    lists = opt_lib._blocked_lists(_dags(3), blocked, None)  # pylint: disable=protected-access
    batch = opt_lib._Batch(_dags(3), True, [0], lists)  # pylint: disable=protected-access
    want = opt_lib._packed_blocked(store, blocked)  # pylint: disable=protected-access
    b = batch.builders[0]
    for dag in b.dags:
        assert b.blocked[dag['blocked_begin']:dag['blocked_end']] == want


def test_change_detection_compares_packed_entries(store):
    """An equal list rebuilt from new Resources objects packs to the same
    entries; another zone, a longer list or another order does not."""
    def key(blocked):
        return opt_lib._entries_key(  # pylint: disable=protected-access
            opt_lib._packed_blocked(store, blocked))  # pylint: disable=protected-access

    a = [_blocked(cloud='aws', region='us-east-1'), _blocked(cloud='gcp')]
    b = [_blocked(cloud='aws', region='us-east-1'), _blocked(cloud='gcp')]
    assert a[0] is not b[0]
    assert key(a) == key(b)
    assert key(a) != key(a[:1])
    assert key(a) != key(a[::-1])
    assert key([]) == key([])
    assert key([_blocked(cloud='aws', region='us-east-1')]) != key(
        [_blocked(cloud='aws', region='us-west-2')])


def test_resolve_dags_symbol_and_signature():
    lib = _native.load()
    assert lib.skyopt_abi_version() == _native.ABI_VERSION
    assert 'skyopt_session_resolve_dags' in _native.EXPORTS
    fn = lib.skyopt_session_resolve_dags
    assert fn.argtypes == [
        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
        ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(_native.Solution),
        ctypes.POINTER(_native.Stats)
    ]
    assert fn.restype is ctypes.c_int
