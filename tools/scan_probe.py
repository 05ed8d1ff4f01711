"""Time the scan kernel alone on a bench workload, in each scan mode named
after the workload (CatalogStore.set_scan_mode; default 'auto')."""
import os
import sys
import numpy as np
sys.path.insert(0, '.')
from skypilot_b200 import workloads as bench  # noqa: E402
import networkx as nx  # noqa: E402
import skypilot_b200 as sky  # noqa: E402
from skypilot_b200 import engine, synth  # noqa: E402
from skypilot_b200 import optimizer as opt_lib  # noqa: E402
from tests import scenario_runner as runner  # noqa: E402

name = sys.argv[1] if len(sys.argv) > 1 else 'cfg4'
w = bench.WORKLOADS[name]
store = sky.catalog.load_frames(synth.make_catalogs(**w['catalog']))
sky.check.set_enabled_clouds(sky.check.ALL_CATALOG_CLOUDS)
dag, tasks = runner.build_dag(bench.chain_scenario(w['tasks']))
O = opt_lib.Optimizer
O._add_dummy_source_sink_nodes(dag)
graph = dag.get_graph()
topo = [t for t in nx.topological_sort(graph) if not opt_lib._is_dummy(t)]
problem = O._state_problem(graph, topo, True, [], True)
for mode in sys.argv[2:] or ['auto']:
    store.set_scan_mode(mode)
    flush = os.environ.get('SKYOPT_NOFLUSH') != '1'  # warm-cache experiment
    engine.solve_timed(problem.builder, 5, flush)
    sol, iter_ms, scan_ms = engine.solve_timed(problem.builder, 30, flush)
    print(name, mode, 'scan_kernel_us', round(1e3 * float(np.mean(scan_ms)), 2),
          'min', round(1e3 * float(np.min(scan_ms)), 2),
          'step_us', round(1e3 * float(np.mean(iter_ms)), 2),
          'blocks', sol.stats.scan_blocks, flush=True)
