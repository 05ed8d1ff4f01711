"""The register-resident chain recurrence (skyopt_step.cuh, lean_recurrence)
and its hazard test, which runs after it from the stored B rows: the fused
step's outputs on both chain paths, a rounding tie crafted to make the hazard
test fire, and chains whose unsatisfiable task is first, in the middle or
last."""
import numpy as np
import pytest

import skypilot_b200 as sky
from skypilot_b200 import engine
from skypilot_b200 import synth
from skypilot_b200 import workloads
from tests import scenario_runner as runner
from tests import scenarios
from tests.test_gpu_chain_handoff import _plan
from tests.test_gpu_chain_handoff import _random_chain
from tests.test_gpu_chain_handoff import _state

pytestmark = pytest.mark.gpu


def _flagship_outputs(workload, mode='auto', path=None):
    """One step of bench.py's device-resident loop on its flagship chain:
    the arrays `bench.py --dump-outputs` writes (engine.Solution, what a
    caller of the device path receives)."""
    store = runner.activate_catalog(workloads.CATALOGS[workload])
    dag, _ = workloads.build_dag(
        workloads.chain_scenario(32 if workload == 'cfg4' else 8))
    builder = engine.ProblemBuilder(store)
    _state(dag, builder)
    with runner.forced_paths(store, mode=mode, chain=path):
        sol, _, _ = engine.solve_timed(builder, 1, True)
    assert sol.dag[0]['status'] == 0
    p = sol.packed
    arrays = {
        'slot_count': sol.slot_count[:p.n_slots],
        'slot_inst': sol.slot_inst[:p.n_slots],
        'chosen_index': sol.chosen_index[:p.n_tasks],
        'task_n_candidates': sol.task_n[:p.n_tasks],
    }
    for prefix, rec, n in (('chosen', sol.chosen, p.n_tasks),
                           ('dag', sol.dag, p.n_dags)):
        for field in rec.dtype.names:
            if not field.endswith('_'):
                arrays[f'{prefix}_{field}'] = rec[field][:n]
    return arrays


@pytest.mark.parametrize('workload', ['cfg2', 'cfg4'])
def test_flagship_chain_same_on_both_chain_paths(workload):
    """cfg2 (8 tasks) and cfg4 (32 tasks): the chain on a block of its own,
    the chain on the block that places the last task and solve_kernel after
    separate launches (scan mode fast-split) give bit-identical outputs."""
    own = _flagship_outputs(workload)
    last = _flagship_outputs(workload, path='32')
    split = _flagship_outputs(workload, mode='fast-split')
    for other in (last, split):
        for name, arr in own.items():
            assert arr.dtype == other[name].dtype
            assert arr.shape == other[name].shape
            assert arr.tobytes() == other[name].tobytes(), name


def _tie(clouds, how='optimize', mode='auto', path=None):
    """A two-task AWS chain. Task 0's instance costs 1e6 an hour, so B of
    task 1 is about 1e6, whose ulp (1.2e-10) swallows 2**-40. Task 1's
    instance costs 1 + 2**-40 in the US regions and 1 elsewhere; AWS lists
    US regions first, so the candidate in front of the cheapest one sums to
    the same double. The reference keeps the first minimum: a US region,
    which only the full evaluation (chain_full) finds, and only if the
    hazard test sends it there. Returns the plan, and the kernel form and
    launches of the call that placed it: Optimizer.optimize's, or a
    session's re-solve (`how` 'session')."""
    frames = synth.make_catalogs(seed=7, n_rows=6000, clouds=clouds.split(','))
    aws = frames['aws']
    big, tied = 'c5.12xlarge', 'c5.2xlarge'
    assert (aws.InstanceType == big).any() and (aws.InstanceType == tied).any()
    aws.loc[aws.InstanceType == big, 'Price'] = 1e6
    us = aws.Region.str.startswith('us-')
    assert (us & (aws.InstanceType == tied)).any()
    assert (~us & (aws.InstanceType == tied)).any()
    aws.loc[(aws.InstanceType == tied) & us, 'Price'] = 1.0 + 2.0 ** -40
    aws.loc[(aws.InstanceType == tied) & ~us, 'Price'] = 1.0
    store = sky.catalog.load_frames(frames)
    sky.check.set_enabled_clouds(sky.check.ALL_CATALOG_CLOUDS)
    sc = workloads.chain('tie', [{'cloud': 'aws', 'instance_type': big},
                                 {'cloud': 'aws', 'instance_type': tied}])
    dag, tasks = workloads.build_dag(sc)
    with runner.forced_paths(store, mode=mode, chain=path):
        if how == 'session':
            with sky.Optimizer.session(dag) as s:
                s.optimize()
                s.optimize([])  # the re-solve: gather_kernel + solve_kernel
                st = s._session.solution.stats  # pylint: disable=protected-access
        else:
            sky.Optimizer.optimize(dag, quiet=True)
            st = engine.LAST_STATS
    return {'plan': [workloads.res_record(t.best_resources) for t in tasks],
            'form': int(st.scan_form), 'launches': int(st.total_launches)}


@pytest.mark.parametrize('clouds', ['aws', 'aws,gcp', 'aws,gcp,azure,lambda'])
def test_rounding_tie_takes_the_first_candidate_on_every_chain_path(clouds):
    """A rounding tie between the cheapest candidate and a pricier one in
    front of it (one, two and four clouds: the three lean loops): the
    default run sends the DAG to the full evaluation and picks the candidate
    in front, as the reference does, equal to the full evaluation forced
    and to the general recurrence forced. So do solve_kernel after separate
    launches (scan mode fast-split) and a session's re-solve under an empty
    blocked list."""
    got = {path: _tie(clouds, path=path) for path in (None, '8', '16')}
    split = _tie(clouds, mode='fast-split')
    resolved = _tie(clouds, how='session')
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
