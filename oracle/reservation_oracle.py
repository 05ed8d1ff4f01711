"""Capacity reservations in the portable oracle: `optimizer_oracle` with the
reference's reservation rules (sky/optimizer.py:259-357).

`run_scenario(catalog_spec, scenario)` runs `optimizer_oracle.run_scenario`
with two of its steps restated for the scenario's `config` and
`reservations` (tests/reservation_scenarios.py):

  * make_launchables_for_valid_region_zones splits AWS per zone when the AWS
    config enables reservations (AWS.optimize_by_zone, aws.py:370-371);
  * _estimate_nodes_cost_or_time prices a candidate at
    `get_cost * max(num_nodes - reserved, 0)`, `reserved` being
    sum(Resources.get_reservations_available_resources().values())
    (resources.py:1785-1812, aws.py:1490-1519, gcp.py:1419-1438).

Everything else (feasibility, region order, DP, totals) is optimizer_oracle's.
"""
import contextlib
from typing import Any, Dict, List

from oracle import optimizer_oracle as oo


def _value(config: Dict[str, Any], cloud: str, key: str, default):
    """<cloud>.<key>: AWS and GCP have no per-region layer in
    get_effective_region_config (config_utils.py:302-330)."""
    return (config.get(cloud) or {}).get(key, default)


def _uses_reservations(config, cloud: str) -> bool:
    """aws_utils.use_reservations (aws_utils.py:30-43); GCP's listing is empty
    under the same condition (gcp_utils.py:141-154)."""
    return bool(_value(config, cloud, 'prioritize_reservations', False) or
                _value(config, cloud, 'specific_reservations', None))


def _need_to_query(config) -> bool:
    """resources_utils.need_to_query_reservations (resources_utils.py:
    425-451)."""
    return any(isinstance(v, dict) and (
        v.get('specific_reservations') is not None or
        v.get('prioritize_reservations')) for v in config.values())


def reserved_nodes(config, inventory, launchable: Dict[str, Any]) -> int:
    if not _need_to_query(config):
        return 0
    cloud = launchable['cloud']
    if (launchable['use_spot'] or launchable.get('zone') is None or
            cloud not in ('aws', 'gcp') or not _uses_reservations(config, cloud)):
        return 0
    names = set(_value(config, cloud, 'specific_reservations', set()) or ())
    by_name = {}  # the reference keeps one count per reservation name
    for r in inventory:
        if (r['cloud'] == cloud and
                r['instance_type'] == launchable['instance_type'] and
                r['zone'] == launchable['zone'] and
                (not r.get('targeted') or r['name'] in names)):
            by_name[r['name']] = r['available']
    return sum(by_name.values())


@contextlib.contextmanager
def _rules(config, inventory):
    saved = oo.make_launchables, oo.estimate_nodes
    aws_by_zone = _uses_reservations(config, 'aws')

    def make_launchables(cat, launchable) -> List[Dict[str, Any]]:
        out = []
        by_zone = launchable['cloud'] == 'gcp' or (
            launchable['cloud'] == 'aws' and aws_by_zone)
        for region, zones in oo.regions_with_offering(cat, launchable):
            if zones is not None and (launchable['use_spot'] or by_zone):
                for zone in zones:
                    out.append(dict(launchable, region=region, zone=zone))
            else:
                out.append(dict(launchable, region=region))
        return out

    def estimate_nodes(cat, tasks, minimize_cost, blocked):
        # optimizer_oracle.estimate_nodes with the reserved nodes subtracted
        tables = []
        for task in tasks:
            filled, fuzzy = oo.fill_in_launchable(cat, task, blocked)
            rows = []
            for req, launch in filled:
                if task.get('time_est') is None:
                    runtime = 1 * 3600
                else:
                    runtime = oo._time_estimator(task['time_est'])(req)  # pylint: disable=protected-access
                for l in launch:
                    if minimize_cost:
                        value = oo.get_cost(cat, l, runtime) * max(
                            task['num_nodes'] -
                            reserved_nodes(config, inventory, l), 0)
                    else:
                        value = runtime
                    rows.append((l, value))
            if not rows:
                raise oo.Unavailable(
                    f'Catalog does not contain any instances satisfying the '
                    f'request: {task["requests"]}. fuzzy={fuzzy}')
            tables.append(rows)
        return tables

    oo.make_launchables, oo.estimate_nodes = make_launchables, estimate_nodes
    try:
        yield
    finally:
        oo.make_launchables, oo.estimate_nodes = saved


def run_scenario(catalog_spec: Dict[str, Any],
                 scenario: Dict[str, Any]) -> Dict[str, Any]:
    """optimizer_oracle.run_scenario under the scenario's reservations."""
    with _rules(scenario.get('config') or {}, scenario.get('reservations', [])):
        return oo.run_scenario(catalog_spec, scenario)
