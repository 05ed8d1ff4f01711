"""Workload for compute-sanitizer: a dozen multi6k scenarios (chains, a
diamond, blocked lists, spot, GCP accelerators) in one kernel mode, plus the
catalog API scan; then one call of each kind that takes temporaries or
session buffers (a list / fuzzy scan, a listing, a non-quiet optimize, a
batch session's open, re-solve and reservation update), and the store's
close, so that --leak-check full sees every buffer freed. The optional
second argument names chain-DP paths to force, comma-separated
engine.set_chain_paths keywords (full, general, last_task_block).

    compute-sanitizer --tool memcheck python tools/sanitize_target.py fast
    compute-sanitizer --tool memcheck python tools/sanitize_target.py auto full
"""
import sys
sys.path.insert(0, '.')
import skypilot_b200 as sky  # noqa: E402
from tests import scenario_runner as runner  # noqa: E402
from tests import scenarios  # noqa: E402
from skypilot_b200 import engine  # noqa: E402
from skypilot_b200 import workloads  # noqa: E402

mode = sys.argv[1] if len(sys.argv) > 1 else 'auto'
chain = sys.argv[2].split(',') if len(sys.argv) > 2 else []
engine.set_chain_paths(**{name: True for name in chain})
payload = runner.load_golden('multi6k')
records = {r['name']: r for r in payload['records']}
store = runner.activate_catalog(payload['catalog'])
store.set_scan_mode(mode)
names = ['acc_V100', 'acc_A100x8', 'cpu_default', 'mem_4x', 'spot_t4x4',
         'chain3_mixed', 'cfg2_chain8', 'cfg3_diamond', 'diamond_time',
         'chain2_egress_big', 'acc_tpu-v3-8', 'cpu_96p']
suite = {s['name']: s for s in scenarios.basic_scenarios()}
bad = 0
for n in names:
    if n not in suite:
        continue
    got = runner.run_scenario(suite[n])
    diffs = runner.compare(records[n], got)
    bad += bool(diffs)
    print(n, 'ok' if not diffs else diffs[:2])

b = engine.ProblemBuilder(store)
for acc, count in (('V100', 1), ('NoSuch', 1)):
    b.add_query(b.accelerator_query('aws', acc, count, want_list=True))
engine.scan(b, list_cap=64, fuzzy_cap=64)
sky.catalog.list_accelerators(all_regions=True)
dag, _ = workloads.build_dag(workloads.chain_scenario(8))
sky.Optimizer.optimize(dag, quiet=False)


def p3_dag():
    with sky.Dag() as d:
        sky.Task('t', num_nodes=4).set_resources(
            sky.Resources(infra='aws', instance_type='p3.2xlarge'))
    return d


def context(available):
    rec = dict(cloud='aws', instance_type='p3.2xlarge', zone='us-west-2b',
               name='cr-q', available=available)
    return sky.PlacementContext(
        enabled_clouds=['aws'], reservations=[rec],
        config={'aws': {'prioritize_reservations': True}})


dags = [p3_dag() for _ in range(3)]
with sky.Optimizer.batch_session(dags, contexts=[context(0)] * 3) as bs:
    bs.optimize()
    bs.optimize([[sky.Resources(infra='aws/us-east-1')], [], []])
    bs.optimize(contexts=[context(0), context(2), context(0)])
store.close()
print('mode', mode, 'chain paths', chain, 'mismatches', bad)
sys.exit(1 if bad else 0)
