"""The chain DP's recovered best parents and its warp-parallel back-track
(at most four clouds) on crafted chains, against oracle/table_dp.py:

* chains of 1, 2, 31 and 32 tasks whose plan changes cloud at every task;
* a parent sum tied bit for bit with another cloud's sum plus a zero tariff,
  the other cloud's candidate first (the smaller id), at the first step with
  parents, a middle step and the sink.
On the default paths and with the full evaluation forced."""
import numpy as np
import pytest

from oracle.table_dp import Tables
from tests import scenario_runner as runner
from tests.test_gpu_dp_tables import _chain_check, _store

pytestmark = pytest.mark.gpu


def alternating(rng, n_tasks, n_clouds):
    """Task t is cheapest in cloud t % n_clouds, egress free."""
    values, clouds = [], []
    for t in range(n_tasks):
        cl = np.concatenate([np.arange(n_clouds), rng.integers(0, n_clouds, 3)])
        rng.shuffle(cl)
        v = np.where(cl == t % n_clouds, 1.0, 2.0 + rng.integers(0, 2, len(cl)))
        values.append(v)
        clouds.append(cl.astype(np.int64))
    zero = np.zeros(n_clouds)
    return Tables(values, clouds, [[t - 1] if t else [] for t in range(n_tasks)],
                  [[zero] if t else [] for t in range(n_tasks)],
                  [None] * n_tasks, n_clouds)


def tied(rng, n_tasks, n_clouds, at):
    """Task `at` - 1 (the last task when `at` == n_tasks: the sink) holds
    equal cheapest values in cloud 1, first, and cloud 0; zero tariffs, so a
    child in cloud 0 sees its own cloud's sum equal to cloud 1's."""
    values, clouds = [], []
    for t in range(n_tasks):
        cl = rng.integers(0, n_clouds, 4)
        v = rng.uniform(2.0, 4.0, 4)
        if t == at - 1:
            cl = np.concatenate([[1, 0], cl])
            v = np.concatenate([[1.0, 1.0], v])
        values.append(v)
        clouds.append(cl.astype(np.int64))
    zero = np.zeros(n_clouds)
    return Tables(values, clouds, [[t - 1] if t else [] for t in range(n_tasks)],
                  [[zero] if t else [] for t in range(n_tasks)],
                  [None] * n_tasks, n_clouds)


def cases():
    for n_clouds in (2, 3, 4):
        for n_tasks in (1, 2, 31, 32):
            rng = np.random.default_rng([n_clouds, n_tasks, 1])
            yield 'alternating', n_clouds, n_tasks, alternating(rng, n_tasks, n_clouds)
        n_tasks = 9
        for at in (1, n_tasks // 2, n_tasks):
            rng = np.random.default_rng([n_clouds, at, 2])
            yield f'tied@{at}', n_clouds, n_tasks, tied(rng, n_tasks, n_clouds, at)


def test_alternating_plans_are_alternating():
    from oracle import table_dp  # pylint: disable=import-outside-toplevel
    for name, n_clouds, n_tasks, tb in cases():
        if name == 'alternating':
            plan, _ = table_dp.chain_dp(tb)
            got = [int(tb.clouds[t][i]) for t, i in enumerate(plan)]
            assert got == [t % n_clouds for t in range(n_tasks)]


@pytest.mark.parametrize('path', [None, '8'])
def test_crafted_chains_match_the_model(path):
    bad, n = [], 0
    stores = {}
    with runner.forced_paths(chain=path):
        for name, n_clouds, n_tasks, tb in cases():
            store = stores.setdefault(n_clouds, _store(n_clouds))
            ok, why = _chain_check(store, tb)
            n += 1
            if not ok:
                bad.append((name, n_clouds, n_tasks, why))
    assert n == 21 and not bad, bad
