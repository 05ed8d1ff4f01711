"""Seeded candidate tables for oracle/table_dp.py and skyopt_solve_tables,
each regime aimed at one way a chain DP or DAG search can go wrong:

  random     magnitudes from 1e-3 to 1e6, tariffs from 0 to 1e3
  quantized  values and tariffs on a coarse grid: exact ties within a cloud
             and across clouds
  hazard     a pricier candidate in front of the cheapest one whose sum rounds
             to the same double (B ~ 1e6 swallows 2^-40): at the first step, a
             middle step, the last step or the sink, in cloud 0 or the last
             cloud, or across two clouds
  sparse     tasks without candidates in some clouds, one cloud without any
  zeros      zero values and zero tariffs, source rows present or absent
  time       TIME-shaped: every value equal and uniform tariffs, so the plan
             is decided by ties alone
  single     tasks of one candidate
  signed     negative values and tariffs, and +-0.0
Candidates of a task are in random cloud order (never sorted by cloud), so
the first minimum in candidate order and the smallest cloud differ.
"""
from typing import Optional

import numpy as np

from oracle.table_dp import Tables

CHAIN_REGIMES = ('random', 'quantized', 'hazard', 'sparse', 'zeros', 'time',
                 'single', 'signed')
_TIE = 2.0 ** -40
_BIG = 1e6


def _row(rng, regime, n_clouds):
    if regime == 'quantized':
        return rng.choice([0.0, 0.25, 0.5], n_clouds)
    if regime == 'zeros':
        return (np.zeros(n_clouds) if rng.random() < 0.5 else
                rng.choice([0.0, 0.5], n_clouds))
    if regime == 'time':
        return np.full(n_clouds, float(rng.choice([0.0, 8.0, 800.0])))
    if regime == 'signed':
        return _signed(rng, n_clouds)
    row = 10.0 ** rng.uniform(-3, 3, n_clouds)
    row[rng.random(n_clouds) < 0.2] = 0.0
    return row


def _signed(rng, n):
    if rng.random() < 0.5:
        # only zeros of both signs and a few small values: a zero objective
        return rng.choice([-0.0, 0.0, 0.5, 1.0], n, p=[0.4, 0.4, 0.1, 0.1])
    x = rng.choice([-1.0, 1.0], n) * 10.0 ** rng.uniform(-3, 3, n)
    z = rng.random(n)
    x[z < 0.15] = -0.0
    x[(z >= 0.15) & (z < 0.3)] = 0.0
    return x


def _values(rng, regime, n):
    if regime == 'quantized':
        return rng.integers(0, 5, n) * 0.25 + 1.0
    if regime == 'zeros':
        return rng.choice([0.0, 0.0, 1.0, 2.5], n)
    if regime == 'time':
        return np.full(n, 3600.0)
    if regime == 'signed':
        return _signed(rng, n)
    return 10.0 ** rng.uniform(-3, 6, n)


def chain(rng, regime: str, n_tasks: int, n_clouds: int,
          empty_at: Optional[int] = None, big_task: Optional[int] = None
          ) -> Tables:
    """A chain of `n_tasks` tasks in `regime`; task `empty_at` without
    candidates, task `big_task` with 10^5."""
    live = list(range(n_clouds))
    if regime == 'sparse' and n_clouds > 1:
        live.remove(int(rng.integers(n_clouds)))   # a cloud nobody has
    # signed: half the chains hold at most one candidate per (task, cloud), so
    # no same-cloud tie sends them to the full evaluation
    distinct = regime == 'signed' and rng.random() < 0.5
    values, clouds, edges, srcs = [], [], [], []
    for t in range(n_tasks):
        n = int(rng.integers(1, 13))
        if regime == 'single' and rng.random() < 0.6:
            n = 1
        if distinct:
            n = min(n, n_clouds)
        if big_task == t:
            n = 100_000
        mine = live
        if regime == 'sparse':
            mine = list(rng.choice(live, int(rng.integers(1, len(live) + 1)),
                                   replace=False))
        if empty_at == t:
            n = 0
        values.append(_values(rng, regime, n))
        clouds.append(rng.choice(mine, n, replace=not distinct).astype(np.int64))
        edges.append([_row(rng, regime, n_clouds)] if t else [])
        srcs.append(_row(rng, regime, n_clouds)
                    if t == 0 and rng.random() < 0.5 else None)
    if regime == 'hazard':
        _plant_hazard(rng, n_tasks, n_clouds, values, clouds, edges, srcs)
    return Tables(values, clouds, [[t - 1] if t else [] for t in
                                   range(n_tasks)], edges, srcs, n_clouds)


def _plant_hazard(rng, n_tasks, n_clouds, values, clouds, edges, srcs):
    """At step s: every parent sum is ~1e6 and the same in every cloud, the
    candidates of one cloud (or of two, `cross`) are the cheapest, and the
    first of them costs 1 + 2^-40, a later one 1: their dp round to the same
    double, so the plan must take the first."""
    s = int(rng.choice([0, n_tasks // 2, max(n_tasks - 2, 0), n_tasks - 1]))
    g = int(rng.choice([0, n_clouds - 1]))
    cross = n_clouds > 1 and rng.random() < 0.35
    if s == 0:
        srcs[0] = np.full(n_clouds, _BIG)
    else:
        values[s - 1] = np.array([_BIG])
        clouds[s - 1] = np.array([int(rng.integers(n_clouds))])
        edges[s] = [np.zeros(n_clouds)]
    n = max(len(values[s]), 2) + 2
    v = rng.uniform(5.0, 50.0, n)
    cl = rng.integers(0, n_clouds, n)
    i = int(rng.integers(0, n - 1))
    j = int(rng.integers(i + 1, n))
    v[i], v[j] = 1.0 + _TIE, 1.0
    if cross:
        cl[i], cl[j] = n_clouds - 1, 0
    else:
        cl[i] = cl[j] = g
        cl[(cl == g) & (np.arange(n) != i) & (np.arange(n) != j)] = (
            (g + 1) % n_clouds) if n_clouds > 1 else g
    values[s], clouds[s] = v, cl.astype(np.int64)
    if s + 1 < n_tasks:
        edges[s + 1] = [np.zeros(n_clouds) if cross else
                        np.full(n_clouds, float(rng.uniform(0, 3)))]


def signed_zero_chains(n_clouds: int):
    """Chains (n_clouds >= 2) where the reference's added zeros decide: every
    source tariff is -0.0, so 0 + src is +0.0 there. (a) Task 0 holds +0.0 in
    cloud 1, then -0.0 in cloud 0; the child in cloud 0 sees equal parent
    sums, and the first candidate wins. (b) 2 and 40 tasks of one -0.0
    candidate each in alternating clouds, -0.0 tariffs: every dp and the
    objective are +0.0."""
    z = np.full(n_clouds, -0.0)
    out = [Tables([[0.0, -0.0], [0.0]], [[1, 0], [0]], [[], [0]],
                  [[], [np.zeros(n_clouds)]], [z, None], n_clouds)]
    for n in (2, 40):
        out.append(Tables([[-0.0]] * n, [[t % 2] for t in range(n)],
                          [[t - 1] if t else [] for t in range(n)],
                          [[z] if t else [] for t in range(n)],
                          [z] + [None] * (n - 1), n_clouds))
    return out


# ---- general DAGs ----------------------------------------------------------
DAG_SHAPES = ('diamond', 'fan', 'random')


def dag_parents(rng, shape: str, n_tasks: int):
    """Parents per task (topological order): a diamond chain, a fan-out into
    a fan-in, or random with one or two parents among the last four."""
    if shape == 'diamond':
        parents = [[]]
        while len(parents) < n_tasks:
            a = len(parents) - 1
            parents.append([a])
            if len(parents) < n_tasks:
                parents.append([a])
            if len(parents) < n_tasks:
                parents.append([len(parents) - 2, len(parents) - 1])
        return parents
    if shape == 'fan':
        mid = list(range(1, n_tasks - 1))
        return [[]] + [[0] for _ in mid] + ([mid or [0]] if n_tasks > 1 else [])
    parents = [[]]
    for j in range(1, n_tasks):
        lo = max(0, j - 4)
        k = min(int(rng.integers(1, 3)), j - lo)
        parents.append(sorted(int(p) for p in rng.choice(range(lo, j), k,
                                                          replace=False)))
    return parents


def dag(rng, regime: str, shape: str, n_tasks: int, n_clouds: int,
        empty_at: Optional[int] = None, options=None) -> Tables:
    """A general DAG with values >= 0. `options[t]`: the number of clouds
    task t has candidates in."""
    parents = dag_parents(rng, shape, n_tasks)
    values, clouds, edges, srcs = [], [], [], []
    for t in range(n_tasks):
        k = options[t] if options is not None else int(
            rng.integers(1, n_clouds + 1))
        mine = rng.choice(n_clouds, k, replace=False)
        n = k + int(rng.integers(0, 6))
        cl = np.concatenate([mine, rng.choice(mine, n - k)])
        rng.shuffle(cl)
        if empty_at == t:
            cl = cl[:0]
        values.append(_values(rng, regime, len(cl)))
        clouds.append(cl.astype(np.int64))
        edges.append([_row(rng, regime, n_clouds) for _ in parents[t]])
        srcs.append(_row(rng, regime, n_clouds)
                    if not parents[t] and rng.random() < 0.5 else None)
    return Tables(values, clouds, parents, edges, srcs, n_clouds)
