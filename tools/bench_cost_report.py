"""cost_report over many cluster records: skypilot_b200.cost_report (one
skyopt_price launch for the whole batch) against the per-record loop of
Resources.get_cost (one device solve per record, two for GCP accelerators),
alternated in one process on the multi50k synthetic catalog.

    python tools/bench_cost_report.py [--sizes 1000 10000 100000] [--reps 2]

Records are seeded (tests/cost_report_cases.random_specs): on-demand and spot,
no region / a region / a zone, GCP hosts with accelerators and TPU VMs, and a
few that cannot be priced. Every total of the two paths must agree bit for
bit. Prints the card and its power limit, then one JSON line per size.
"""
import argparse
import json
import logging
import os
import subprocess
import sys
import time

_REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, _REPO)

import skypilot_b200 as sky  # pylint: disable=wrong-import-position
from tests import cost_report_cases as cases  # pylint: disable=wrong-import-position
from tests import scenario_runner as runner  # pylint: disable=wrong-import-position
from tests import scenarios  # pylint: disable=wrong-import-position


def _loop(records):
    out = []
    for record in records:
        report = record.copy()
        try:
            report['total_cost'] = (record['resources'].get_cost(
                record['duration']) * record['num_nodes'])
        except Exception:  # pylint: disable=broad-except
            report['total_cost'] = 0.0
        out.append(report)
    return out


def _card() -> str:
    return subprocess.run(
        ['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
        capture_output=True, text=True, check=True).stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', type=int, nargs='+',
                    default=[1000, 10000, 100000])
    ap.add_argument('--reps', type=int, default=2)
    args = ap.parse_args()
    logging.disable(logging.WARNING)  # the failing records' warnings
    print('card:', _card(), flush=True)
    spec = scenarios.CATALOGS['multi50k']
    runner.activate_catalog(spec)
    frames = cases.catalog_frames(spec)
    warm = cases.history(cases.random_specs(frames, 200, seed=1))
    sky.cost_report(warm)
    _loop(warm)
    for n in args.sizes:
        records = cases.history(cases.random_specs(frames, n, seed=n))
        t_batch, t_loop = [], []
        batch = loop = None
        for _ in range(args.reps):
            t0 = time.perf_counter()
            batch = sky.cost_report(records)
            t_batch.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            loop = _loop(records)
            t_loop.append(time.perf_counter() - t0)
        same = all(
            a['total_cost'] == b['total_cost'] or
            (a['total_cost'] != a['total_cost'] and
             b['total_cost'] != b['total_cost']) for a, b in zip(batch, loop))
        if not same:
            raise SystemExit(f'{n} records: totals differ')
        failed = sum(r['total_cost'] == 0.0 for r in batch)
        print(json.dumps({
            'records': n, 'zero_or_failed': failed,
            'cost_report_s': min(t_batch), 'get_cost_loop_s': min(t_loop),
            'speedup': min(t_loop) / min(t_batch), 'totals_agree': same,
            'card': _card()
        }), flush=True)


if __name__ == '__main__':
    main()
