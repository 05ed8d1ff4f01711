"""The AWS account's zone mapping without a GPU: the oracle against the
reference's records on the mapped `azmap` catalog, what the ingest keeps and
drops, the choice of the mapping file, the catalog cache key, and the host
statement on the mapped catalog."""
import hashlib
import json
import os

import numpy as np
import pandas as pd
import pytest

from oracle import azmap_oracle
from oracle import optimizer_oracle as oo
from skypilot_b200 import synth
from skypilot_b200.catalog import store as store_lib
from skypilot_b200.catalog.store import CatalogStore
from tests import azmap_runner
from tests import azmap_scenarios
from tests import scenario_runner as runner
from tests.test_host_statement import _stated_instances


@pytest.fixture(scope='module')
def frames_mapping():
    return azmap_scenarios.frames_and_mapping()


@pytest.fixture(scope='module')
def mapped_store():
    return azmap_runner.build_store()


def _gold():
    return dict(azmap_runner.records('azmap'),
                **azmap_runner.records('azmap_reservations'))


@pytest.mark.parametrize('scenario', azmap_runner.optimizer_scenarios(),
                         ids=lambda s: s['name'])
def test_oracle_reproduces_reference_record(scenario):
    gold = _gold()[scenario['name']]
    if gold.get('error', {}).get('type') == 'ValueError':
        # rejected while the request is built (a zone ID, a region the
        # account lacks), like Resources() in the reference
        with pytest.raises(ValueError):
            azmap_oracle.run_scenario(azmap_scenarios.CATALOG,
                                      azmap_scenarios.AZ_MAPPING_SEED,
                                      scenario)
        return
    got = azmap_oracle.run_scenario(azmap_scenarios.CATALOG,
                                    azmap_scenarios.AZ_MAPPING_SEED, scenario)
    if 'error' in gold:
        # the oracle words infeasibility itself; the device tests compare
        # the reference's text
        assert 'error' in got, got
        return
    assert 'error' not in got, got['error']
    assert got['candidates'] == gold['candidates']
    assert got['plan'] == gold['plan']
    assert runner.close(got['objective'], gold['objective'])
    if gold['is_chain']:
        assert got['objective'] == gold['objective']
    assert runner.close(got['total_cost'], gold['total_cost'])
    assert runner.close(got['total_time'], gold['total_time'])


def test_fixture_plans_name_only_mapped_zones(frames_mapping):
    _, mapping = frames_mapping
    names = set(mapping['AvailabilityZoneName'])
    unmapped = set(azmap_scenarios.UNMAPPED_REGIONS)
    n_zoned = 0
    for rec in _gold().values():
        for p in rec.get('plan', []):
            if p['cloud'] == 'aws':
                assert p['region'] not in unmapped, rec['name']
                if p['zone'] is not None:
                    assert p['zone'] in names, (rec['name'], p['zone'])
                    n_zoned += 1
        for cands in rec.get('candidates', []):
            for c in cands:
                if c[0] == 'aws':
                    assert c[2] not in unmapped
                    assert c[3] is None or c[3] in names
    assert n_zoned > 0
    errors = {n: r['error']['message'] for n, r in _gold().items()
              if 'error' in r}
    assert 'use1-az3' in errors['zone_id_rejected']
    assert 'eu-west-2' in errors['unmapped_region']


def test_generated_mapping_has_the_promised_shape(frames_mapping):
    frames, mapping = frames_mapping
    aws = frames['aws']
    by_region = {}
    for name, zid in zip(mapping['AvailabilityZoneName'],
                         mapping['AvailabilityZone']):
        by_region.setdefault(name[:-1], []).append((zid, name))
    ids = aws.groupby('Region')['AvailabilityZone'].nunique()
    assert set(azmap_scenarios.UNMAPPED_REGIONS) == set(ids.index) - set(
        by_region)
    partly = [r for r, pairs in by_region.items() if len(pairs) < ids[r]]
    assert len(partly) == 3
    for region, pairs in by_region.items():
        pairs.sort()
        if len(pairs) > 1:
            # name order differs from ID order in every region
            assert [n for _, n in pairs] != sorted(n for _, n in pairs)
    # the zone-ID style changes nothing else, and is opt-in
    plain = synth.make_catalogs(**dict(azmap_scenarios.CATALOG,
                                       aws_zone_ids=False))
    assert plain['aws'].drop(columns='AvailabilityZone').equals(
        aws.drop(columns='AvailabilityZone'))
    assert all(z.startswith(r) for z, r in zip(
        plain['aws']['AvailabilityZone'], plain['aws']['Region']))
    for cloud in ('gcp', 'runpod'):
        assert plain[cloud].equals(frames[cloud])


def test_ingest_drops_unmapped_rows_and_ranks_by_name(frames_mapping,
                                                      mapped_store):
    frames, mapping = frames_mapping
    aws = frames['aws']
    to_name = dict(zip(mapping['AvailabilityZone'],
                       mapping['AvailabilityZoneName']))
    kept = aws[aws['AvailabilityZone'].isin(to_name)]
    table = mapped_store.cloud('aws')
    assert table.n_rows == len(kept) < len(aws)
    assert table.region_names == sorted(set(kept['Region']))
    for region in azmap_scenarios.UNMAPPED_REGIONS:
        assert region not in table.region_exact
    assert table.zone_names == sorted(set(mapping['AvailabilityZoneName']) &
                                      set(kept['AvailabilityZone'].map(
                                          to_name)))
    assert not any(z in table.zone_exact for z in to_name)
    cols = mapped_store.columns
    rows = slice(table.row_begin, table.row_end)
    zone_of_row = [table.zone_names[z] for z in cols['zone_id'][rows]]
    region_of_row = [table.region_names[r] for r in cols['region_id'][rows]]
    # rows keep the catalog's order; ranks are name ranks
    assert zone_of_row == list(kept['AvailabilityZone'].map(to_name))
    assert region_of_row == list(kept['Region'])
    for z, name in enumerate(table.zone_names):
        assert table.region_names[table.zone_region[z]] == name[:-1]
    # the other clouds are untouched
    plain = CatalogStore.from_frames(frames)
    for cloud in ('gcp', 'runpod'):
        a, b = plain.cloud(cloud), mapped_store.cloud(cloud)
        assert (a.region_names, a.zone_names, a.n_rows) == (
            b.region_names, b.zone_names, b.n_rows)


def _aws_frame():
    return pd.DataFrame({
        'InstanceType': ['m6i.large', 'm6i.large', 'm6i.large', 'm6i.large'],
        'vCPUs': [2.0] * 4, 'MemoryGiB': [8.0] * 4,
        'Price': [0.1, 0.1, 0.2, 0.2], 'SpotPrice': [0.03, 0.04, 0.05, 0.06],
        'Region': ['us-east-1', 'us-east-1', 'us-west-2', 'us-west-2'],
        'AvailabilityZone': ['use1-az1', 'use1-az2', 'usw2-az1', 'usw2-az2'],
    })


def _mapping(pairs):
    return pd.DataFrame(pairs,
                        columns=['AvailabilityZoneName', 'AvailabilityZone'])


def test_merge_follows_the_reference():
    df = store_lib.apply_az_mapping(_aws_frame(), _mapping(
        [('us-east-1b', 'use1-az1'), ('us-east-1a', 'use1-az2'),
         ('us-west-2a', 'usw2-az2'), ('eu-west-1a', 'euw1-az1')]))
    assert list(df['AvailabilityZone']) == ['us-east-1b', 'us-east-1a',
                                            'us-west-2a']
    assert list(df['SpotPrice']) == [0.03, 0.04, 0.06]
    assert 'AvailabilityZoneName' not in df.columns


@pytest.mark.parametrize('pairs,message', [
    ([('us-east-1a', 'use1-az1'), ('us-east-1b', 'use1-az1')],
     "zone ID 'use1-az1' is mapped to 2 values"),
    ([('us-east-1a', 'use1-az1'), ('us-east-1a', 'use1-az2')],
     "zone name 'us-east-1a' is mapped to 2 values"),
])
def test_malformed_mapping_is_rejected(pairs, message):
    with pytest.raises(ValueError, match=message):
        CatalogStore.from_frames({'aws': _aws_frame()},
                                 aws_az_mapping=_mapping(pairs))


def test_mapping_without_its_columns_is_rejected():
    bad = pd.DataFrame({'ZoneName': ['us-east-1a'], 'ZoneId': ['use1-az1']})
    with pytest.raises(ValueError, match='missing columns'):
        CatalogStore.from_frames({'aws': _aws_frame()}, aws_az_mapping=bad)
    # a duplicated identical pair is not a conflict
    ok = _mapping([('us-east-1a', 'use1-az1'), ('us-east-1a', 'use1-az1')])
    store = CatalogStore.from_frames({'aws': _aws_frame()}, aws_az_mapping=ok)
    assert store.cloud('aws').zone_names == ['us-east-1a']


def _catalog_dir(tmp_path, files):
    os.makedirs(tmp_path / 'aws', exist_ok=True)
    _aws_frame().to_csv(tmp_path / 'aws' / 'vms.csv', index=False)
    for i, (name, pairs) in enumerate(files):
        path = tmp_path / 'aws' / f'az_mappings-{name}.csv'
        _mapping(pairs).to_csv(path, index=False)
        os.utime(path, (1_600_000_000 + i, 1_600_000_000 + i))
    return str(tmp_path)


_OLD = [('us-east-1a', 'use1-az1'), ('us-east-1b', 'use1-az2')]
_NEW = [('us-east-1c', 'use1-az1'), ('us-west-2c', 'usw2-az1')]


def test_hash_names_the_file_and_newest_wins_without_one(tmp_path):
    path = _catalog_dir(tmp_path, [('aaaa1111', _OLD), ('bbbb2222', _NEW)])
    assert store_lib.find_az_mapping(path, 'aaaa1111').endswith(
        'az_mappings-aaaa1111.csv')
    assert store_lib.find_az_mapping(path).endswith('az_mappings-bbbb2222.csv')
    assert store_lib.find_az_mapping(path, 'cccc3333') is None
    by_hash = CatalogStore.from_directory(path, use_cache=False,
                                          aws_user_hash='aaaa1111')
    assert by_hash.cloud('aws').zone_names == ['us-east-1a', 'us-east-1b']
    newest = CatalogStore.from_directory(path, use_cache=False)
    assert newest.cloud('aws').zone_names == ['us-east-1c', 'us-west-2c']
    # an account without its file keeps the zone IDs
    unknown = CatalogStore.from_directory(path, use_cache=False,
                                          aws_user_hash='cccc3333')
    assert unknown.cloud('aws').zone_names == ['use1-az1', 'use1-az2',
                                               'usw2-az1', 'usw2-az2']


def _cache_keys(path):
    return set(os.listdir(os.path.join(path, '.skyopt_cache')))


def test_cache_key_covers_the_mapping_file(tmp_path):
    path = _catalog_dir(tmp_path / 'plain', [])
    CatalogStore.from_directory(path)
    st = os.stat(os.path.join(path, 'aws', 'vms.csv'))
    unchanged = hashlib.sha256(json.dumps(
        [store_lib.CACHE_VERSION,
         [['aws', st.st_size, st.st_mtime_ns]]]).encode()).hexdigest()[:24]
    assert _cache_keys(path) == {unchanged}

    path = _catalog_dir(tmp_path / 'mapped', [('aaaa1111', _OLD)])
    first = CatalogStore.from_directory(path)
    keys = _cache_keys(path)
    assert len(keys) == 1
    warm = CatalogStore.from_directory(path)
    assert _cache_keys(path) == keys
    assert warm.cloud('aws').zone_names == first.cloud('aws').zone_names
    mapping = os.path.join(path, 'aws', 'az_mappings-aaaa1111.csv')
    _mapping(_NEW).to_csv(mapping, index=False)
    os.utime(mapping, (1_700_000_000, 1_700_000_000))
    touched = CatalogStore.from_directory(path)
    assert len(_cache_keys(path)) == 2
    assert touched.cloud('aws').zone_names == ['us-east-1c', 'us-west-2c']


def test_load_frames_with_mapping_equals_load_directory(tmp_path,
                                                        frames_mapping,
                                                        mapped_store):
    frames, mapping = frames_mapping
    for cloud, frame in frames.items():
        os.makedirs(tmp_path / cloud)
        frame.to_csv(tmp_path / cloud / 'vms.csv', index=False)
    mapping.to_csv(tmp_path / 'aws' / 'az_mappings-0a1b2c3d.csv', index=False)
    loaded = CatalogStore.from_directory(str(tmp_path), clouds=list(frames),
                                         use_cache=False,
                                         aws_user_hash='0a1b2c3d')
    for name, col in mapped_store.columns.items():
        other = loaded.columns[name]
        if col is None:
            assert other is None, name
        else:
            np.testing.assert_array_equal(col, other, err_msg=name)
    for a, b in zip(mapped_store.clouds, loaded.clouds):
        assert (a.name, a.region_names, a.zone_names, a.zone_region,
                a.inst_names) == (b.name, b.region_names, b.zone_names,
                                  b.zone_region, b.inst_names)


def _statement_cases():
    return [s for s in azmap_scenarios.azmap_scenarios()
            if all(t.get('resources_kind', 'single') == 'single'
                   for t in s['tasks'])]


@pytest.mark.parametrize('scenario', _statement_cases(),
                         ids=lambda s: s['name'])
def test_stated_queries_pick_the_oracles_instance(scenario):
    store = azmap_runner.activate()
    cat = oo.catalog_for(azmap_oracle._spec(  # pylint: disable=protected-access
        azmap_scenarios.CATALOG, azmap_scenarios.AZ_MAPPING_SEED))
    try:
        got = _stated_instances(store, scenario)
    except ValueError:
        # requests rejected while they are built (a zone ID, an unmapped
        # region): the oracle rejects them too
        with pytest.raises(ValueError):
            for tspec in scenario['tasks']:
                oo.normalize_request(cat, tspec['resources'][0])
        return
    for ti, tspec in enumerate(scenario['tasks']):
        req = oo.normalize_request(cat, tspec['resources'][0])
        clouds = [req['cloud']] if req['cloud'] is not None else cat.enabled
        for cloud in clouds:
            launchables, _ = oo.feasible(cat, cloud, dict(req, cloud=cloud),
                                         tspec.get('num_nodes', 1))
            if not launchables:
                continue
            assert got.get((ti, 0, cloud)) == launchables[0]['instance_type'], (
                ti, cloud)
