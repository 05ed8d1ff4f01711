"""Exact model of `skyopt_solve_tables` on candidate tables -- test
infrastructure (only tests/ import this).

Inputs as for `engine.solve_tables`: per task the candidate values and their
clouds, the parents, a tariff row per parent (indexed by the parent's cloud)
and an optional source row (indexed by the task's cloud).

* Chains: the reference's `_optimize_by_dp` (sky/optimizer.py:429-487)
  operation by operation: `0 + src[c]`, `dp[p] + (0 if same cloud else
  tar[cloud_p])`, strict `<` (the first minimum in candidate order), `value +
  best`, sink `dp + 0`, objective `0 + best`. `chain_dp` takes the minimum
  per child cloud with numpy's first-occurrence argmin; `chain_dp_loop` is
  the literal per-candidate loop.
* General DAGs: the exact optimum over one representative per (task, cloud),
  COST summed with math.fsum (frontier_dp beyond an enumeration limit), TIME
  by the reference's finish-time recursion (`_compute_total_time`).
"""
import itertools
import math
import operator
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from oracle import dag_oracle


class Tables:
    """One DAG's candidate tables, in the layout of engine.solve_tables."""

    def __init__(self, values, clouds, parents, edge_tariffs, src_tariffs,
                 n_clouds: int):
        self.values = [np.asarray(v, dtype=np.float64) for v in values]
        self.clouds = [np.asarray(c, dtype=np.int64) for c in clouds]
        self.parents = [list(p) for p in parents]
        self.edge_tariffs = [[np.asarray(r, dtype=np.float64) for r in rows]
                             for rows in edge_tariffs]
        self.src_tariffs = [None if s is None else np.asarray(s, np.float64)
                            for s in src_tariffs]
        self.n_clouds = n_clouds

    @property
    def n_tasks(self) -> int:
        return len(self.values)

    def args(self):
        """Positional arguments of engine.solve_tables after the store."""
        return ([v.tolist() for v in self.values],
                [c.tolist() for c in self.clouds], self.parents,
                [[r.tolist() for r in rows] for rows in self.edge_tariffs],
                [None if s is None else s.tolist() for s in self.src_tariffs])

    def first_empty(self) -> Optional[int]:
        for t, v in enumerate(self.values):
            if len(v) == 0:
                return t
        return None


def chain_dp(tb: Tables) -> Tuple[List[int], float]:
    """(chosen index per task, objective) of the reference's chain DP."""
    dp = back = None
    for t in range(tb.n_tasks):
        v, cl = tb.values[t], tb.clouds[t]
        if t == 0:
            src = tb.src_tariffs[0]
            best = 0.0 + (src[cl] if src is not None else np.zeros(len(v)))
            ptr = np.zeros(len(v), dtype=np.int64)
        else:
            tar = tb.edge_tariffs[t][0]
            pcl = tb.clouds[t - 1]
            best = np.empty(len(v))
            ptr = np.empty(len(v), dtype=np.int64)
            for h in np.unique(cl):
                sums = dp + np.where(pcl == h, 0.0, tar[pcl])
                i = int(np.argmin(sums))
                best[cl == h] = sums[i]
                ptr[cl == h] = i
        dp, back = v + best, (back or []) + [ptr]
    sink = dp + 0.0
    idx = int(np.argmin(sink))
    objective = 0.0 + float(sink[idx])
    plan = [0] * tb.n_tasks
    for t in range(tb.n_tasks - 1, -1, -1):
        plan[t] = idx
        idx = int(back[t][idx])
    return plan, objective


def chain_dp_loop(tb: Tables, take=operator.lt, sink_take=operator.lt,
                  same_cloud_egress: bool = False) -> Tuple[List[int], float]:
    """chain_dp as the reference writes it: every (child, parent) pair. The
    keyword arguments plant the bugs tests/test_table_dp.py shows its table
    regimes expose (`<=` for `take`, egress on same-cloud edges, ...)."""
    dp: List[List[float]] = []
    back: List[List[int]] = []
    for t in range(tb.n_tasks):
        cur, ptr = [], []
        for c in range(len(tb.values[t])):
            cc = int(tb.clouds[t][c])
            best, best_p = math.inf, -1
            if t == 0:
                src = tb.src_tariffs[0]
                v = 0 + (float(src[cc]) if src is not None else 0)
                if v < best:
                    best, best_p = v, 0
            else:
                tar = tb.edge_tariffs[t][0]
                for p, pv in enumerate(dp[t - 1]):
                    cp = int(tb.clouds[t - 1][p])
                    v = pv + (float(tar[cp]) if same_cloud_egress or cp != cc
                              else 0)
                    if take(v, best):
                        best, best_p = v, p
            cur.append(float(tb.values[t][c]) + best)
            ptr.append(best_p)
        dp.append(cur)
        back.append(ptr)
    best, idx = math.inf, -1
    for p, v in enumerate(dp[-1]):
        if sink_take(v + 0, best):
            best, idx = v + 0, p
    plan = [0] * tb.n_tasks
    for t in range(tb.n_tasks - 1, -1, -1):
        plan[t] = idx
        idx = back[t][idx]
    return plan, 0 + best


# ---- general DAGs ----------------------------------------------------------
def representatives(tb: Tables) -> List[Dict[int, int]]:
    """Per task {cloud: first candidate of the smallest value in it}."""
    reps = []
    for v, cl in zip(tb.values, tb.clouds):
        r: Dict[int, int] = {}
        for i in range(len(v)):
            c = int(cl[i])
            if c not in r or v[i] < v[r[c]]:
                r[c] = i
        reps.append(r)
    return reps


def _egress(tb: Tables, t: int, k: int, cp: int, cc: int) -> float:
    return 0.0 if cp == cc else float(tb.edge_tariffs[t][k][cp])


def _src(tb: Tables, t: int, cc: int) -> float:
    src = tb.src_tariffs[t]
    return 0.0 if tb.parents[t] or src is None else float(src[cc])


def dag_objective(tb: Tables, chosen: Sequence[int],
                  minimize_cost: bool) -> float:
    """The objective of a plan (one candidate index per task): COST as an
    exact sum, TIME as the reference's finish time of the dummy sink (with
    values and tariffs >= 0, the largest finish time of any task)."""
    cl = [int(tb.clouds[t][i]) for t, i in enumerate(chosen)]
    if minimize_cost:
        terms = []
        for t, i in enumerate(chosen):
            terms.append(float(tb.values[t][i]))
            terms.append(_src(tb, t, cl[t]))
            for k, p in enumerate(tb.parents[t]):
                terms.append(_egress(tb, t, k, cl[p], cl[t]))
        return math.fsum(terms)
    finish: List[float] = []
    for t, i in enumerate(chosen):
        starts = [0, 0 + _src(tb, t, cl[t])]
        for k, p in enumerate(tb.parents[t]):
            starts.append(finish[p] + _egress(tb, t, k, cl[p], cl[t]))
        finish.append(float(tb.values[t][i]) + max(starts))
    children = {p for ps in tb.parents for p in ps}
    return 0 + max([0] + [finish[t] + 0 for t in range(tb.n_tasks)
                          if t not in children])


def dag_optimum(tb: Tables, minimize_cost: bool,
                enumerate_limit: int = 20000) -> Tuple[float, List[int]]:
    """(exact optimum, one optimal plan) of a general DAG."""
    reps = representatives(tb)
    n_assign = math.prod(len(r) for r in reps)
    if n_assign <= enumerate_limit:
        best, plan = math.inf, None
        for combo in itertools.product(*[sorted(r.values()) for r in reps]):
            obj = dag_objective(tb, combo, minimize_cost)
            if obj < best:
                best, plan = obj, list(combo)
        return best, plan
    assert minimize_cost, 'TIME: enumeration only'
    order = list(range(tb.n_tasks))
    children = {t: [] for t in order}
    for t, ps in enumerate(tb.parents):
        for p in ps:
            children[p].append(t)
    parents = {t: tb.parents[t] for t in order}
    options = {t: sorted(r.values()) for t, r in enumerate(reps)}

    def node_cost(t, i):
        return float(tb.values[t][i]) + _src(tb, t, int(tb.clouds[t][i]))

    def edge_cost(p, ip, t, i):
        k = tb.parents[t].index(p)
        return _egress(tb, t, k, int(tb.clouds[p][ip]), int(tb.clouds[t][i]))

    best, plan = dag_oracle.frontier_dp(order, children, parents, options,
                                        node_cost, edge_cost)
    chosen = [plan[t] for t in order]
    return dag_objective(tb, chosen, True), chosen
