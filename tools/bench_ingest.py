"""Catalog ingest: CSV parse + SoA build vs the columnar cache (host CPU
only, no GPU involved; SURVEY.md section 8f rank 1). Prints one JSON line per
catalog size and AWS zone style: the catalog as generated, and the same
catalog with AWS zone IDs plus an account's `aws/az_mappings-*.csv`, which
the ingest merges before encoding (CatalogStore.from_directory)."""
import json
import os
import sys
import tempfile
import time

sys.path.insert(0, '.')
from skypilot_b200 import workloads as bench  # noqa: E402
from skypilot_b200 import synth  # noqa: E402
from skypilot_b200.catalog.store import CatalogStore  # noqa: E402


def measure(name: str, az_mapping: bool) -> dict:
    spec = dict(bench.WORKLOADS[name]['catalog'])
    if az_mapping:
        spec['aws_zone_ids'] = True
    frames = synth.make_catalogs(**spec)
    with tempfile.TemporaryDirectory() as d:
        for cloud, df in frames.items():
            os.makedirs(os.path.join(d, cloud))
            df.to_csv(os.path.join(d, cloud, 'vms.csv'), index=False)
        if az_mapping:
            synth.aws_az_mapping(frames['aws'], spec['seed']).to_csv(
                os.path.join(d, 'aws', 'az_mappings-0a1b2c3d.csv'),
                index=False)
        t0 = time.perf_counter()
        a = CatalogStore.from_directory(d, use_cache=False)
        t1 = time.perf_counter()
        CatalogStore.from_directory(d)          # parses and writes the cache
        t2 = time.perf_counter()
        CatalogStore.from_directory(d)          # cache hit
        t3 = time.perf_counter()
        CatalogStore.from_directory(d)          # cache hit, warm imports
        t4 = time.perf_counter()
        size = sum(os.path.getsize(os.path.join(r, f))
                   for r, _, fs in os.walk(os.path.join(d, '.skyopt_cache'))
                   for f in fs)
        csv = sum(os.path.getsize(os.path.join(d, c, 'vms.csv')) for c in frames)
    return {'catalog': name, 'aws_az_mapping': az_mapping, 'device': 'host CPU',
            'rows': int(a.n_real_rows),
            'csv_parse_and_ingest_s': round(t1 - t0, 3),
            'parse_ingest_and_save_s': round(t2 - t1, 3),
            'cache_load_first_s': round(t3 - t2, 3),
            'cache_load_s': round(t4 - t3, 3),
            'csv_bytes': csv, 'cache_bytes': size}


for catalog in sys.argv[1:] or ['cfg2', 'cfg4']:
    for mapped in (False, True):
        print(json.dumps(measure(catalog, mapped)))
