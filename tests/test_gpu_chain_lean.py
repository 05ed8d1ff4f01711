"""The register-resident chain recurrence (skyopt_step.cuh, lean_recurrence)
and its hazard test, which runs after it from the stored B rows: the fused
step's outputs on both chain paths, a rounding tie crafted to make the hazard
test fire, and chains whose unsatisfiable task is first, in the middle or
last. The SKYOPT_EXP knobs are read once per process, hence the
subprocesses."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from skypilot_b200 import engine
from skypilot_b200 import workloads
from tests import scenario_runner as runner
from tests import scenarios
from tests.test_gpu_chain_handoff import _plan
from tests.test_gpu_chain_handoff import _random_chain
from tests.test_gpu_chain_handoff import _state

pytestmark = pytest.mark.gpu

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(args, exp):
    env = dict(os.environ)
    env.pop('SKYOPT_EXP', None)
    if exp:
        env['SKYOPT_EXP'] = exp
    proc = subprocess.run([sys.executable] + args, cwd=_ROOT, env=env,
                          capture_output=True, text=True, timeout=900,
                          check=False)
    assert proc.returncode == 0, proc.stdout[-2000:] + proc.stderr[-2000:]
    return proc.stdout


def _bench_outputs(workload, exp, out_dir, split=False):
    _run(['bench.py', '--no-extras', '--steps', '1', '--warmup', '0',
          '--workload', workload, '--dump-outputs', out_dir] +
         (['--scan-mode', 'fast-split'] if split else []), exp)
    return {
        f: np.load(os.path.join(out_dir, f))
        for f in sorted(os.listdir(out_dir)) if f.endswith('.npy')
    }


@pytest.mark.parametrize('workload', ['cfg2', 'cfg4'])
def test_flagship_chain_same_on_both_chain_paths(workload):
    """cfg2 (8 tasks) and cfg4 (32 tasks): the chain on a block of its own,
    the chain on the block that places the last task (SKYOPT_EXP=32) and
    solve_kernel after separate launches (scan mode fast-split) give
    bit-identical outputs."""
    with tempfile.TemporaryDirectory() as tmp:
        own = _bench_outputs(workload, None, os.path.join(tmp, 'own'))
        last = _bench_outputs(workload, '32', os.path.join(tmp, 'last'))
        split = _bench_outputs(workload, None, os.path.join(tmp, 'split'),
                               split=True)
    assert own and sorted(own) == sorted(last) == sorted(split)
    for other in (last, split):
        for name, arr in own.items():
            assert arr.dtype == other[name].dtype
            assert arr.shape == other[name].shape
            assert arr.tobytes() == other[name].tobytes(), name


# A two-task AWS chain. Task 0's instance costs 1e6 an hour, so B of task 1
# is about 1e6, whose ulp (1.2e-10) swallows 2**-40. Task 1's instance costs
# 1 + 2**-40 in the US regions and 1 elsewhere; AWS lists US regions first,
# so the candidate in front of the cheapest one sums to the same double. The
# reference keeps the first minimum: a US region, which only the full
# evaluation (chain_full) finds, and only if the hazard test sends it there.
_TIE_SCRIPT = r'''
import json, sys
sys.path.insert(0, ".")
import skypilot_b200 as sky
from skypilot_b200 import engine, synth, workloads
clouds = sys.argv[1].split(",")
frames = synth.make_catalogs(seed=7, n_rows=6000, clouds=clouds)
aws = frames["aws"]
big, tied = "c5.12xlarge", "c5.2xlarge"
assert (aws.InstanceType == big).any() and (aws.InstanceType == tied).any()
aws.loc[aws.InstanceType == big, "Price"] = 1e6
us = aws.Region.str.startswith("us-")
assert (us & (aws.InstanceType == tied)).any() and (~us & (aws.InstanceType == tied)).any()
aws.loc[(aws.InstanceType == tied) & us, "Price"] = 1.0 + 2.0 ** -40
aws.loc[(aws.InstanceType == tied) & ~us, "Price"] = 1.0
store = sky.catalog.load_frames(frames)
sky.check.set_enabled_clouds(sky.check.ALL_CATALOG_CLOUDS)
sc = workloads.chain("tie", [{"cloud": "aws", "instance_type": big},
                             {"cloud": "aws", "instance_type": tied}])
dag, tasks = workloads.build_dag(sc)
if sys.argv[3] == "split":
    store.set_scan_mode("fast-split")
if sys.argv[2] == "session":
    with sky.Optimizer.session(dag) as s:
        s.optimize()
        s.optimize([])  # the re-solve: gather_kernel + solve_kernel
        st = s._session.solution.stats
else:
    sky.Optimizer.optimize(dag, quiet=True)
    st = engine.LAST_STATS
print(json.dumps({"plan": [workloads.res_record(t.best_resources) for t in tasks],
                  "form": int(st.scan_form), "launches": int(st.total_launches)}))
'''


@pytest.mark.parametrize('clouds', ['aws', 'aws,gcp', 'aws,gcp,azure,lambda'])
def test_rounding_tie_takes_the_first_candidate_on_every_chain_path(clouds):
    """A rounding tie between the cheapest candidate and a pricier one in
    front of it (one, two and four clouds: the three lean loops): the
    default run sends the DAG to the full evaluation and picks the candidate
    in front, as the reference does, equal to the full evaluation forced
    (SKYOPT_EXP=8) and to the general recurrence (SKYOPT_EXP=16). So do
    solve_kernel after separate launches (scan mode fast-split) and a
    session's re-solve under an empty blocked list."""
    def run(exp=None, split=False, how='optimize'):
        out = _run(['-c', _TIE_SCRIPT, clouds, how,
                    'split' if split else 'auto'], exp)
        return json.loads(out.strip().splitlines()[-1])

    got = {exp: run(exp) for exp in (None, '8', '16')}
    split = run(split=True)
    resolved = run(how='session')
    assert got[None]['form'] == 4
    assert split['form'] == 3
    assert resolved['form'] == 0 and resolved['launches'] == 2
    assert got[None]['plan'] == got['8']['plan'] == got['16']['plan']
    assert got[None]['plan'] == split['plan'] == resolved['plan']
    second = got[None]['plan'][1]
    assert second['instance_type'] == 'c5.2xlarge'
    assert second['region'].startswith('us-'), second


def _empty_at(name, n, k):
    """An n-task chain whose task k nothing satisfies."""
    specs = [{'accelerators': 'V100', 'outputs_gb': 20} for _ in range(n)]
    specs[k] = {'cpus': '100000+'}
    return workloads.chain(name, specs)


def test_unsatisfiable_task_first_middle_last_in_one_launch():
    """Chains whose unsatisfiable task is the first, a middle or the last
    one, with satisfiable chains between them, in one fused launch: each
    reports the first such task, and the others equal the same DAG solved
    alone."""
    store = runner.activate_catalog(scenarios.CATALOGS['multi6k'])
    rng = np.random.default_rng(5)
    chains = [
        _empty_at('e_first', 6, 0), _random_chain(rng, 'a'),
        _empty_at('e_mid', 7, 3), _random_chain(rng, 'b'),
        _empty_at('e_last', 5, 4), _random_chain(rng, 'c'),
    ]
    fail_at = {'e_first': 0, 'e_mid': 3, 'e_last': 4}
    batch = engine.ProblemBuilder(store)
    sizes = []
    for sc in chains:
        dag, tasks = workloads.build_dag(sc)
        _state(dag, batch)
        sizes.append(len(tasks))
    sol = engine.solve(batch)
    stats = engine.LAST_STATS
    assert int(stats.scan_form) == 4 and int(stats.total_launches) == 1
    first = 0
    for i, (sc, n) in enumerate(zip(chains, sizes)):
        got = _plan(sol, first, n, i)
        if sc['name'] in fail_at:
            assert got == {'status': 1, 'task_fail': fail_at[sc['name']]}
        else:
            one = engine.ProblemBuilder(store)
            dag, _ = workloads.build_dag(sc)
            _state(dag, one)
            assert got == _plan(engine.solve(one), 0, n, 0), sc['name']
            assert got['status'] == 0
        first += n
