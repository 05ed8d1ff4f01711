"""Catalog ingest: per-cloud `vms.csv` frames -> structure-of-arrays in HBM.

Replaces the reference's pandas catalog (`read_catalog` / `LazyDataFrame`,
sky/catalog/common.py:126-266): the CSV columns are dictionary-encoded once,
per-cloud Python rules become flag bits (rules.py), and the result is uploaded
to the GPU through `skyopt_catalog_create`. Everything the kernels scan lives
in ten columns (32 B per row and pass, see DESIGN.md):

  price, spot_price, vcpus, mem : f64   (NaN = missing, as in pandas)
  acc_key    : u16  id of the (AcceleratorName, AcceleratorCount) pair
  region_id  : u16  rank of Region among the cloud's region names
  zone_id    : u16  rank of AvailabilityZone (0xFFFF = missing)
  flags      : u16  SKYOPT_F_* bits | instance group << 8
  (+ inst_id i32 and disk_total f64, gathered only for matching rows)

Ranks are taken in Python string order, which is the order pandas sorts the
object columns in (`sort_values(['Price', 'Region', 'AvailabilityZone'])`,
common.py:797-802), so comparing ids on the device equals comparing names.
Row order inside a cloud is the CSV order; "cheapest" ties resolve to the
lowest row id (the reference's single-key sort is unstable, SURVEY.md).
"""
import ctypes
import glob
import hashlib
import json
import os
import threading
import weakref
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import pandas as pd

from skypilot_b200 import _native
from skypilot_b200.catalog import rules as rules_lib

_ROW_ALIGN = _native.ZONE_ROWS  # clouds start on a zone-map boundary
CATALOG_SCHEMA_VERSION = 'v8'


def _col(df: pd.DataFrame, name: str, n: int) -> np.ndarray:
    if name in df.columns:
        return pd.to_numeric(df[name], errors='coerce').to_numpy(
            dtype=np.float64, na_value=np.nan)
    return np.full(n, np.nan)


def price_keys(values: np.ndarray) -> np.ndarray:
    """Order-preserving double -> uint64 map (skyopt_price_key in C): flip
    the sign bit of non-negative values, all bits of negative ones."""
    bits = np.ascontiguousarray(values, dtype=np.float64).view(np.uint64)
    neg = (bits >> np.uint64(63)).astype(bool)
    return np.where(neg, ~bits, bits | np.uint64(1 << 63))


CACHE_VERSION = 2  # layout + ingest rules of the columnar cache written by CatalogStore.save
# (2: per-cloud frame filters and preferred regions are applied at ingest)

AZ_MAPPING_COLUMNS = ('AvailabilityZoneName', 'AvailabilityZone')


def apply_az_mapping(aws: pd.DataFrame, mapping: pd.DataFrame) -> pd.DataFrame:
    """The AWS account's zone mapping applied to the AWS catalog, as
    sky/catalog/aws_catalog.py:179-185 does: an inner merge on the zone ID
    (rows in zones or regions the account lacks are dropped), the ID column
    dropped and the account's zone name renamed to AvailabilityZone.

    The mapping comes from outside the program (`aws/az_mappings-*.csv`), so
    it is checked first: a zone ID mapped to two names would duplicate rows,
    and a name reached from two IDs would break one row per (InstanceType,
    AvailabilityZone) and zone names unique across regions
    (sky/catalog/common.py:355, :385)."""
    missing = [c for c in AZ_MAPPING_COLUMNS if c not in mapping.columns]
    if missing:
        raise ValueError(f'AWS zone mapping: missing columns {missing}; a '
                         f'mapping has {list(AZ_MAPPING_COLUMNS)}')
    if 'AvailabilityZone' not in aws.columns:
        raise ValueError('AWS zone mapping: the AWS catalog has no '
                         'AvailabilityZone column')
    pairs = mapping[list(AZ_MAPPING_COLUMNS)].drop_duplicates()
    for key, other in (('AvailabilityZone', 'AvailabilityZoneName'),
                       ('AvailabilityZoneName', 'AvailabilityZone')):
        dup = pairs[pairs[key].duplicated(keep=False)]
        if len(dup):
            first = dup[key].iloc[0]
            values = sorted(str(v) for v in dup[dup[key] == first][other])
            what = 'zone ID' if key == 'AvailabilityZone' else 'zone name'
            raise ValueError(f'AWS zone mapping: {what} {first!r} is mapped '
                             f'to {len(values)} values {values}')
    df = aws.merge(pairs, on=['AvailabilityZone'], how='inner')
    return df.drop(columns=['AvailabilityZone']).rename(
        columns={'AvailabilityZoneName': 'AvailabilityZone'})


def find_az_mapping(path: str,
                    aws_user_hash: Optional[str] = None) -> Optional[str]:
    """The mapping file the reference would read below a catalog directory
    (sky/catalog/aws_catalog.py:94-117, :142-168): with the account's hash
    `aws/az_mappings-<hash>.csv` if it exists; without one the most recently
    modified `aws/az_mappings-*.csv`. None: keep the zone IDs."""
    if aws_user_hash is not None:
        name = os.path.join(path, 'aws', f'az_mappings-{aws_user_hash}.csv')
        return name if os.path.exists(name) else None
    files = glob.glob(os.path.join(glob.escape(path), 'aws',
                                   'az_mappings-*.csv'))
    if not files:
        return None
    files.sort(key=os.path.getmtime)
    return files[-1]


def _zone_map(cols: Dict[str, np.ndarray]) -> np.ndarray:
    """Static summary of every 128-row chunk: flag bits and accelerator keys
    (mod 64) that occur, fixed-host groups (mod 32), cheapest Price / SpotPrice. The scan kernel tests a
    query against the summary before it touches the chunk's rows."""
    zr = _native.ZONE_ROWS
    n = len(cols['flags'])
    assert n % zr == 0
    nz = n // zr
    flags = cols['flags'].reshape(nz, zr)
    valid = (flags & _native.F_VALID) != 0
    zone = np.zeros(nz, dtype=_native.ZONE_DTYPE)
    zone['flags_or'] = np.bitwise_or.reduce(
        np.where(valid, flags & 0xFF, 0).astype(np.uint32), axis=1)
    ak = cols['acc_key'].reshape(nz, zr).astype(np.uint64)
    has = valid & (ak != _native.NONE16)
    sig = np.bitwise_or.reduce(
        np.where(has, np.uint64(1) << (ak & np.uint64(63)), np.uint64(0)),
        axis=1)
    zone['sig_lo'] = (sig & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    zone['sig_hi'] = (sig >> np.uint64(32)).astype(np.uint32)
    grp = (flags >> 8).astype(np.uint32)
    zone['groups'] = np.bitwise_or.reduce(
        np.where(valid & (grp != 0), np.uint32(1) << (grp & np.uint32(31)),
                 np.uint32(0)), axis=1)
    none = np.uint64(0xFFFFFFFFFFFFFFFF)
    for c, name in enumerate(('price', 'spot_price')):
        p = cols[name].reshape(nz, zr)
        ok = valid & ~np.isnan(p)
        keys = np.where(ok, price_keys(np.nan_to_num(p, nan=0.0)), none)
        zone['min_key'][:, c] = keys.min(axis=1)
    return zone


class CloudTable:
    """Host-side dictionaries and metadata of one cloud."""

    def __init__(self, name: str, index: int):
        self.name = name
        self.index = index
        self.rules = rules_lib.rules_for(name)
        self.row_begin = 0
        self.row_end = 0  # exclusive, without padding
        self.n_rows = 0
        self.region_names: List[str] = []
        self.region_lower: Dict[str, int] = {}
        self.region_exact: Dict[str, int] = {}
        self.zone_names: List[str] = []
        self.zone_lower: Dict[str, int] = {}
        self.zone_exact: Dict[str, int] = {}
        self.zone_region: List[int] = []
        self.has_zone_column = False
        self.inst_begin = 0
        self.inst_names: List[str] = []
        self.inst_index: Dict[str, int] = {}  # name -> GLOBAL id
        self.frame: Optional[pd.DataFrame] = None  # original rows (metadata)
        self.inst_first_row: Optional[np.ndarray] = None  # local row ids
        # summary of the 'GpuInfo' column (accelerator listings): None = no
        # such column
        self.gpu_info_any_nan = False
        self.gpu_info_unique: Optional[List[str]] = []


class CatalogStore:
    """All enabled clouds' catalogs as one SoA table (+ the device handle)."""

    def __init__(self):
        self.clouds: List[CloudTable] = []
        self.cloud_index: Dict[str, int] = {}
        self.acc_keys: List[Tuple[str, float]] = []
        self.acc_key_index: Dict[Tuple[str, float], int] = {}
        self.acc_names_lower: List[str] = []
        self.inst_names: List[str] = []
        self.inst_cloud: List[int] = []
        self.columns: Dict[str, np.ndarray] = {}
        self.n_rows = 0  # padded
        self.n_real_rows = 0
        self.max_group_rows = 1
        self._handles: Dict[int, ctypes.c_void_p] = {}
        self._lock = threading.Lock()
        self._keepalive: List[np.ndarray] = []
        self._sessions = weakref.WeakSet()  # open engine.Session objects
        # <cloud>/images.csv (Tag, Region, ImageId, ...): a few rows, host only
        self.images: Dict[str, pd.DataFrame] = {}
        # common/metadata.csv (GPU, MemoryGB, Manufacturer): '32GB+' requests
        self.metadata: Optional[pd.DataFrame] = None

    # ------------------------------------------------------------------ build
    @classmethod
    def from_frames(cls,
                    frames: Dict[str, pd.DataFrame],
                    order: Optional[Sequence[str]] = None,
                    aws_az_mapping: Optional[pd.DataFrame] = None
                    ) -> 'CatalogStore':
        """`aws_az_mapping` (AvailabilityZoneName, AvailabilityZone rows) is
        applied to the AWS frame before anything is encoded
        (`apply_az_mapping`), so ranks, zone map and orders are the mapped
        catalog's."""
        store = cls()
        names = list(order) if order is not None else list(frames.keys())
        if aws_az_mapping is not None and 'aws' in names:
            frames = dict(frames,
                          aws=apply_az_mapping(frames['aws'], aws_az_mapping))
        if len(names) > _native.MAX_CLOUDS:
            raise ValueError(f'at most {_native.MAX_CLOUDS} clouds')
        price, spot, vcpus, mem, disk = [], [], [], [], []
        acc_key, region_id, zone_id, flags, inst_id = [], [], [], [], []
        cloud_row_offsets = [0]
        cloud_inst_offsets = [0]
        cloud_region_offsets = [0]
        cloud_n_zones = []
        region_is_us: List[int] = []
        any_disk = False
        for ci, name in enumerate(names):
            df = frames[name].reset_index(drop=True)
            table = CloudTable(name, ci)
            if table.rules.frame_filter is not None:
                # the cloud's catalog module filters its CSV when loading it
                df = table.rules.frame_filter(df).reset_index(drop=True)
            table.frame = df
            n = len(df)
            if 'GpuInfo' in df.columns:
                info = df['GpuInfo']
                table.gpu_info_any_nan = bool(info.isna().any())
                table.gpu_info_unique = [str(t) for t in info.dropna().unique()]
            else:
                table.gpu_info_unique = None
            table.n_rows = n
            table.row_begin = cloud_row_offsets[-1]
            table.row_end = table.row_begin + n
            rules = table.rules
            # --- instance types: first-appearance order
            it = df['InstanceType'] if 'InstanceType' in df.columns else (
                pd.Series([None] * n, dtype=object))
            codes, uniques = pd.factorize(it, use_na_sentinel=True)
            table.inst_names = [str(u) for u in uniques]
            table.inst_begin = cloud_inst_offsets[-1]
            table.inst_index = {
                nm: table.inst_begin + i
                for i, nm in enumerate(table.inst_names)
            }
            gl_inst = np.where(codes >= 0, codes + table.inst_begin,
                               -1).astype(np.int32)
            first_row = np.full(len(uniques), -1, dtype=np.int64)
            if n:
                order_idx = np.arange(n)
                valid = codes >= 0
                # first occurrence per code
                rev = order_idx[valid][::-1]
                first_row[codes[valid][::-1]] = rev
            table.inst_first_row = first_row
            store.inst_names.extend(table.inst_names)
            store.inst_cloud.extend([ci] * len(table.inst_names))
            cloud_inst_offsets.append(table.inst_begin + len(uniques))
            # --- regions / zones: ranks in string order
            reg = df['Region'].astype(object)
            table.region_names = sorted(str(r) for r in reg.dropna().unique())
            rmap = {nm: i for i, nm in enumerate(table.region_names)}
            table.region_exact = dict(rmap)
            for nm, i in rmap.items():
                low = nm.lower()
                if low in table.region_lower:
                    raise ValueError(
                        f'{name}: regions {nm!r} and '
                        f'{table.region_names[table.region_lower[low]]!r} '
                        'differ only in case')
                table.region_lower[low] = i
            if len(table.region_names) >= _native.NONE16:
                raise ValueError(f'{name}: too many regions')
            if reg.isna().any():
                raise ValueError(f'{name}: rows without a Region')
            rid = reg.map(rmap).to_numpy(dtype=np.int64).astype(np.uint16)
            table.has_zone_column = 'AvailabilityZone' in df.columns
            zid = np.full(n, _native.NONE16, dtype=np.uint16)
            if table.has_zone_column:
                zone = df['AvailabilityZone'].astype(object)
                table.zone_names = sorted(
                    str(z) for z in zone.dropna().unique())
                if len(table.zone_names) >= _native.NONE16:
                    raise ValueError(f'{name}: too many zones')
                zmap = {nm: i for i, nm in enumerate(table.zone_names)}
                table.zone_exact = dict(zmap)
                table.zone_lower = {nm.lower(): i for nm, i in zmap.items()}
                has = zone.notna().to_numpy()
                zid[has] = zone[has].map(zmap).to_numpy(dtype=np.int64)
                zr = np.full(len(table.zone_names), -1, dtype=np.int64)
                zr[zid[has]] = rid[has]
                table.zone_region = [int(v) for v in zr]
            cloud_region_offsets.append(cloud_region_offsets[-1] +
                                        len(table.region_names))
            cloud_n_zones.append(
                max(len(table.zone_names), 1) if table.has_zone_column else 0)
            preferred = rules.preferred_region or (
                lambda name: name.startswith('us-'))
            region_is_us.extend(
                1 if preferred(r) else 0 for r in table.region_names)
            # --- accelerators: (name, count) dictionary over all clouds
            ak = np.full(n, _native.NONE16, dtype=np.uint16)
            if 'AcceleratorName' in df.columns:
                an = df['AcceleratorName'].astype(object)
                ac = _col(df, 'AcceleratorCount', n)
                has = an.notna().to_numpy() & ~np.isnan(ac)
                if has.any():
                    pairs = pd.MultiIndex.from_arrays(
                        [an[has].astype(str).to_numpy(), ac[has]])
                    pcodes, puniq = pd.factorize(pairs)
                    ids = np.empty(len(puniq), dtype=np.int64)
                    for j, (nm, cnt) in enumerate(puniq):
                        key = (str(nm), float(cnt))
                        if key not in store.acc_key_index:
                            store.acc_key_index[key] = len(store.acc_keys)
                            store.acc_keys.append(key)
                        ids[j] = store.acc_key_index[key]
                    ak[has] = ids[pcodes]
            # --- flags from the per-cloud rules (once per instance type)
            per_inst = np.zeros(len(uniques), dtype=np.uint16)
            for j, nm in enumerate(table.inst_names):
                f = _native.F_HAS_INSTANCE
                if rules.default_family is None or rules.default_family(nm):
                    f |= _native.F_DEFAULT_FAMILY
                if rules.host_family is not None and rules.host_family(nm):
                    f |= _native.F_HOST_FAMILY
                if rules.premium_disk is not None:
                    try:
                        if rules.premium_disk(nm):
                            f |= _native.F_PREMIUM_DISK
                    except ValueError:
                        pass
                if rules.group_of is not None:
                    f |= (rules.group_of(nm) & 0xFF) << 8
                per_inst[j] = f
            fl = np.full(n, _native.F_VALID, dtype=np.uint16)
            has_inst = codes >= 0
            fl[has_inst] |= per_inst[codes[has_inst]]
            if rules.default_family is None:
                # clouds without a default-family rule search the whole frame
                fl |= _native.F_DEFAULT_FAMILY
            dt = np.zeros(n, dtype=np.float64)
            if 'LocalDiskType' in df.columns:
                any_disk = True
                ssd = (df['LocalDiskType'] == 'ssd').to_numpy(dtype=bool)
                fl[ssd] |= _native.F_SSD
                if 'NVMeSupported' in df.columns:
                    nv = df['NVMeSupported']
                    nvme = (nv == True).to_numpy(dtype=bool)  # pylint: disable=singleton-comparison
                    fl[nvme] |= _native.F_NVME
                size = np.nan_to_num(_col(df, 'LocalDiskSize', n), nan=0.0)
                cnt = np.nan_to_num(_col(df, 'LocalDiskCount', n), nan=0.0)
                dt = size * cnt
            # --- pad to the row alignment
            pad = (-n) % _ROW_ALIGN

            def padded(arr, fill):
                if pad == 0:
                    return arr
                return np.concatenate(
                    [arr, np.full(pad, fill, dtype=arr.dtype)])

            price.append(padded(_col(df, 'Price', n), np.nan))
            spot.append(padded(_col(df, 'SpotPrice', n), np.nan))
            vcpus.append(padded(_col(df, 'vCPUs', n), np.nan))
            mem.append(padded(_col(df, 'MemoryGiB', n), np.nan))
            disk.append(padded(dt, 0.0))
            acc_key.append(padded(ak, _native.NONE16))
            region_id.append(padded(rid, 0))
            zone_id.append(padded(zid, _native.NONE16))
            flags.append(padded(fl, 0))
            inst_id.append(padded(gl_inst, -1))
            cloud_row_offsets.append(cloud_row_offsets[-1] + n + pad)
            store.clouds.append(table)
            store.cloud_index[name] = ci
            store.n_real_rows += n
        if len(store.acc_keys) > 32 * _native.ACC_SET_WORDS:
            raise ValueError('too many distinct (accelerator, count) pairs')
        cols = store.columns
        cols['price'] = np.ascontiguousarray(np.concatenate(price))
        cols['spot_price'] = np.ascontiguousarray(np.concatenate(spot))
        cols['vcpus'] = np.ascontiguousarray(np.concatenate(vcpus))
        cols['mem'] = np.ascontiguousarray(np.concatenate(mem))
        cols['disk_total'] = (np.ascontiguousarray(np.concatenate(disk))
                              if any_disk else None)
        cols['acc_key'] = np.ascontiguousarray(np.concatenate(acc_key))
        cols['region_id'] = np.ascontiguousarray(np.concatenate(region_id))
        cols['zone_id'] = np.ascontiguousarray(np.concatenate(zone_id))
        cols['flags'] = np.ascontiguousarray(np.concatenate(flags))
        cols['inst_id'] = np.ascontiguousarray(np.concatenate(inst_id))
        store.n_rows = int(cloud_row_offsets[-1])
        cols['cloud_row_offsets'] = np.asarray(cloud_row_offsets, np.int32)
        cols['cloud_inst_offsets'] = np.asarray(cloud_inst_offsets, np.int32)
        cols['cloud_region_offsets'] = np.asarray(cloud_region_offsets,
                                                  np.int32)
        cols['cloud_n_zones'] = np.asarray(cloud_n_zones, np.int32)
        cols['region_is_us'] = np.asarray(region_is_us or [0], np.uint8)
        store._finish_columns()
        return store

    def _finish_columns(self) -> None:
        """Derived side tables of the per-row columns: the CSR of rows per
        instance type / accelerator key and the zone map."""
        store, cols = self, self.columns
        # --- CSR: rows grouped by instance type (ascending row order inside)
        iid = cols['inst_id']
        n_inst = len(store.inst_names)
        rows = np.flatnonzero(iid >= 0).astype(np.int32)
        order_idx = np.argsort(iid[rows], kind='stable')
        cols['inst_rows'] = np.ascontiguousarray(rows[order_idx])
        counts = np.bincount(iid[rows], minlength=n_inst)
        cols['inst_row_offsets'] = np.concatenate(
            [[0], np.cumsum(counts)]).astype(np.int32)
        # accelerator-only rows (GCP GPU / TPU rows) grouped by key
        n_keys = len(store.acc_keys)
        akc = cols['acc_key']
        arow = np.flatnonzero((iid < 0) & (akc != _native.NONE16) &
                              ((cols['flags'] & _native.F_VALID) != 0)).astype(
                                  np.int32)
        aorder = np.argsort(akc[arow], kind='stable')
        cols['acc_rows'] = np.ascontiguousarray(arow[aorder])
        acounts = np.bincount(akc[arow].astype(np.int64), minlength=n_keys)
        cols['acc_row_offsets'] = np.concatenate(
            [[0], np.cumsum(acounts)]).astype(np.int32)
        iak = np.full(max(n_inst, 1), _native.NONE16, dtype=np.uint16)
        if n_inst:
            firsts = cols['inst_rows'][cols['inst_row_offsets'][:-1].clip(
                max=max(len(cols['inst_rows']) - 1, 0))]
            nonempty = counts > 0
            iak[:n_inst][nonempty] = akc[firsts[nonempty]]
        cols['inst_acc_key'] = iak
        cols['zone_map'] = _zone_map(cols)
        store.max_group_rows = int(
            max([1] + list(counts) + list(acounts)))
        store.acc_names_lower = [k[0].lower() for k in store.acc_keys]

    _ROW_COLUMNS = (('price', np.nan), ('spot_price', np.nan),
                    ('vcpus', np.nan), ('mem', np.nan), ('disk_total', 0.0),
                    ('acc_key', _native.NONE16), ('region_id', 0),
                    ('zone_id', _native.NONE16), ('flags', 0), ('inst_id', -1))

    def replicated(self, k: int) -> 'CatalogStore':
        """A catalog with every cloud's rows repeated `k` times (same names,
        same dictionaries): a larger-than-L2 table for the HBM stress row of
        bench.py. Equal prices resolve to the lowest row, so every answer is
        the original catalog's answer -- which the bench checks."""
        import copy  # pylint: disable=import-outside-toplevel
        new = CatalogStore()
        new.acc_keys = list(self.acc_keys)
        new.acc_key_index = dict(self.acc_key_index)
        new.inst_names = list(self.inst_names)
        new.inst_cloud = list(self.inst_cloud)
        new.cloud_index = dict(self.cloud_index)
        parts: Dict[str, List[np.ndarray]] = {n: [] for n, _ in
                                              self._ROW_COLUMNS}
        offsets = [0]
        for table in self.clouds:
            t = copy.copy(table)
            n = table.n_rows * k
            pad = (-n) % _ROW_ALIGN
            for name, fill in self._ROW_COLUMNS:
                col = self.columns.get(name)
                if col is None:
                    continue
                real = np.tile(col[table.row_begin:table.row_end], k)
                if pad:
                    real = np.concatenate(
                        [real, np.full(pad, fill, dtype=real.dtype)])
                parts[name].append(real)
            t.row_begin = offsets[-1]
            t.n_rows = n
            t.row_end = t.row_begin + n
            offsets.append(offsets[-1] + n + pad)
            new.clouds.append(t)
            new.n_real_rows += n
        for name, _ in self._ROW_COLUMNS:
            new.columns[name] = (np.ascontiguousarray(
                np.concatenate(parts[name])) if parts[name] else None)
        for name in ('cloud_inst_offsets', 'cloud_region_offsets',
                     'cloud_n_zones', 'region_is_us'):
            new.columns[name] = self.columns[name]
        new.columns['cloud_row_offsets'] = np.asarray(offsets, np.int32)
        new.n_rows = int(offsets[-1])
        new._finish_columns()  # pylint: disable=protected-access
        return new

    @classmethod
    def from_directory(cls,
                       path: str,
                       clouds: Optional[Sequence[str]] = None,
                       use_cache: bool = True,
                       aws_user_hash: Optional[str] = None) -> 'CatalogStore':
        """Loads `<path>/<cloud>/vms.csv` (the reference's on-disk layout,
        sky/catalog/common.py:33-35, :65-68).

        The AWS catalog lists zone IDs; the account's
        `aws/az_mappings-*.csv` that `find_az_mapping` picks for
        `aws_user_hash` turns them into its zone names and drops what the
        account cannot use (`apply_az_mapping`).

        The parsed catalog is kept next to the CSVs as a columnar binary cache
        (`<path>/.skyopt_cache/<key>/`, see `save`): the reference re-parses
        the CSVs in every process (`pd.read_csv` behind LazyDataFrame,
        common.py:126-164, ~1.5 s for the public catalog); a warm start here
        maps the same columns that are uploaded to the GPU. The key covers the
        files' names, sizes and modification times, so an edited or refreshed
        CSV is parsed again."""
        path = os.path.expanduser(path)
        names = clouds
        if names is None:
            names = sorted(
                d for d in os.listdir(path)
                if os.path.exists(os.path.join(path, d, 'vms.csv')))
        files = [(name, os.path.join(path, name, 'vms.csv')) for name in names]
        files = [(name, csv) for name, csv in files if os.path.exists(csv)]
        if not files:
            raise FileNotFoundError(f'no <cloud>/vms.csv below {path}')
        mapping_csv = (find_az_mapping(path, aws_user_hash)
                       if any(name == 'aws' for name, _ in files) else None)
        cache_dir = None
        if use_cache:
            sig = []
            for name, csv in files:
                st = os.stat(csv)
                sig.append([name, st.st_size, st.st_mtime_ns])
            if mapping_csv is not None:
                # without a mapping file the key is what it always was
                st = os.stat(mapping_csv)
                sig.append([os.path.join('aws', os.path.basename(mapping_csv)),
                            st.st_size, st.st_mtime_ns])
            key = hashlib.sha256(
                json.dumps([CACHE_VERSION, sig]).encode()).hexdigest()[:24]
            cache_dir = os.path.join(path, '.skyopt_cache', key)
            if os.path.exists(os.path.join(cache_dir, 'meta.json')):
                try:
                    store = cls.load(cache_dir)
                    store.load_images(path)
                    return store
                except Exception:  # pylint: disable=broad-except
                    # unreadable / corrupt cache (zipfile.BadZipFile, a
                    # truncated parquet, ...): parse the CSVs again
                    import shutil  # pylint: disable=import-outside-toplevel
                    shutil.rmtree(cache_dir, ignore_errors=True)
        frames = {name: pd.read_csv(csv) for name, csv in files}
        mapping = (pd.read_csv(mapping_csv) if mapping_csv is not None else
                   None)
        store = cls.from_frames(frames, order=list(frames.keys()),
                                aws_az_mapping=mapping)
        store.load_images(path)
        if cache_dir is not None:
            try:
                store.save(cache_dir)
            except OSError:
                pass  # read-only catalog directory: stay uncached
        return store

    # ------------------------------------------------------ columnar cache
    def save(self, directory: str) -> None:
        """Writes the catalog as a columnar binary cache: `columns.npz` (the
        SoA columns exactly as they are uploaded, zone map included),
        `meta.json` (dictionaries: region / zone / instance-type names,
        accelerator keys) and `types_<cloud>.parquet` (one CSV row per
        instance type, for metadata look-ups)."""
        # Everything is written into a private scratch directory and committed
        # with ONE rename: two processes ingesting the same catalog at once
        # cannot interleave their files, and a reader never sees a half-written
        # cache. Whoever renames first wins; the loser drops its copy.
        import shutil  # pylint: disable=import-outside-toplevel
        import uuid  # pylint: disable=import-outside-toplevel
        final = directory.rstrip(os.sep)
        os.makedirs(os.path.dirname(final) or '.', exist_ok=True)
        directory = f'{final}.tmp.{os.getpid()}.{uuid.uuid4().hex[:8]}'
        os.makedirs(directory)
        try:
            self._write_cache_files(directory)
            try:
                os.rename(directory, final)  # commit point
            except OSError:
                if not os.path.exists(os.path.join(final, 'meta.json')):
                    raise
        finally:
            if os.path.isdir(directory):
                shutil.rmtree(directory, ignore_errors=True)

    def _write_cache_files(self, directory: str) -> None:
        arrays = {k: v for k, v in self.columns.items() if v is not None}
        np.savez(os.path.join(directory, 'columns.npz'), **arrays)
        meta = {
            'version': CACHE_VERSION, 'n_rows': self.n_rows,
            'n_real_rows': self.n_real_rows,
            'max_group_rows': self.max_group_rows,
            'acc_keys': [[n, c] for n, c in self.acc_keys],
            'inst_cloud': self.inst_cloud, 'clouds': []
        }
        for t in self.clouds:
            rows = t.inst_first_row
            types = t.frame.iloc[np.where(rows >= 0, rows, 0)].reset_index(
                drop=True)
            types.to_parquet(os.path.join(directory, f'types_{t.name}.parquet'))
            meta['clouds'].append({
                'name': t.name, 'row_begin': t.row_begin, 'row_end': t.row_end,
                'n_rows': t.n_rows, 'region_names': t.region_names,
                'zone_names': t.zone_names, 'zone_region': t.zone_region,
                'has_zone_column': t.has_zone_column,
                'inst_begin': t.inst_begin, 'inst_names': t.inst_names,
                'inst_has_row': [bool(r >= 0) for r in rows],
                'gpu_info_any_nan': t.gpu_info_any_nan,
                'gpu_info_unique': t.gpu_info_unique,
            })
        with open(os.path.join(directory, 'meta.json'), 'w',
                  encoding='utf-8') as f:
            json.dump(meta, f)

    @classmethod
    def load(cls, directory: str) -> 'CatalogStore':
        """Inverse of `save`: no CSV parsing, no per-row work."""
        with open(os.path.join(directory, 'meta.json'), encoding='utf-8') as f:
            meta = json.load(f)
        if meta.get('version') != CACHE_VERSION:
            raise ValueError('catalog cache version mismatch')
        store = cls()
        with np.load(os.path.join(directory, 'columns.npz')) as data:
            for k in data.files:
                store.columns[k] = np.ascontiguousarray(data[k])
        store.columns.setdefault('disk_total', None)
        store.n_rows = int(meta['n_rows'])
        store.n_real_rows = int(meta['n_real_rows'])
        store.max_group_rows = int(meta['max_group_rows'])
        store.acc_keys = [(str(n), float(c)) for n, c in meta['acc_keys']]
        store.acc_key_index = {k: i for i, k in enumerate(store.acc_keys)}
        store.acc_names_lower = [k[0].lower() for k in store.acc_keys]
        store.inst_cloud = [int(c) for c in meta['inst_cloud']]
        for ci, m in enumerate(meta['clouds']):
            t = CloudTable(m['name'], ci)
            t.row_begin, t.row_end = int(m['row_begin']), int(m['row_end'])
            t.n_rows = int(m['n_rows'])
            t.region_names = list(m['region_names'])
            t.region_exact = {nm: i for i, nm in enumerate(t.region_names)}
            t.region_lower = {nm.lower(): i
                              for i, nm in enumerate(t.region_names)}
            t.zone_names = list(m['zone_names'])
            t.zone_exact = {nm: i for i, nm in enumerate(t.zone_names)}
            t.zone_lower = {nm.lower(): i for i, nm in enumerate(t.zone_names)}
            t.zone_region = [int(v) for v in m['zone_region']]
            t.has_zone_column = bool(m['has_zone_column'])
            t.inst_begin = int(m['inst_begin'])
            t.inst_names = list(m['inst_names'])
            t.inst_index = {nm: t.inst_begin + i
                            for i, nm in enumerate(t.inst_names)}
            t.frame = pd.read_parquet(
                os.path.join(directory, f'types_{t.name}.parquet'))
            has_row = np.asarray(m['inst_has_row'], dtype=bool)
            t.inst_first_row = np.where(has_row, np.arange(len(has_row)),
                                        -1).astype(np.int64)
            t.gpu_info_any_nan = bool(m['gpu_info_any_nan'])
            t.gpu_info_unique = m['gpu_info_unique']
            store.inst_names.extend(t.inst_names)
            store.clouds.append(t)
            store.cloud_index[t.name] = ci
        return store

    # --------------------------------------------------------------- look-ups
    def cloud(self, name: str) -> CloudTable:
        return self.clouds[self.cloud_index[name.lower()]]

    def has_cloud(self, name: str) -> bool:
        return name.lower() in self.cloud_index

    def instance_id(self, cloud: str, instance_type: str) -> int:
        return self.cloud(cloud).inst_index.get(instance_type, -1)

    def instance_row(self, cloud: str, instance_type: str) -> pd.Series:
        """First CSV row of an instance type (metadata look-ups)."""
        table = self.cloud(cloud)
        gid = table.inst_index.get(instance_type)
        if gid is None:
            raise KeyError(instance_type)
        return table.frame.iloc[int(
            table.inst_first_row[gid - table.inst_begin])]

    def accelerator_set(self, predicate) -> np.ndarray:
        """Bitmask (ACC_SET_WORDS u32) of the keys `predicate(name, count)`."""
        words = np.zeros(_native.ACC_SET_WORDS, dtype=np.uint32)
        for k, (name, count) in enumerate(self.acc_keys):
            if predicate(name, count):
                words[k >> 5] |= np.uint32(1 << (k & 31))
        return words

    def accelerator_name_clouds(self) -> Dict[str, set]:
        """{accelerator name: clouds offering it} (the role of the
        reference's common/accelerators.csv)."""
        cached = getattr(self, '_acc_name_clouds', None)
        if cached is not None:
            return cached
        out: Dict[str, set] = {}
        akc = self.columns['acc_key']
        offsets = self.columns['cloud_row_offsets']
        for ci, table in enumerate(self.clouds):
            keys = np.unique(akc[offsets[ci]:offsets[ci + 1]])
            for k in keys:
                if k != _native.NONE16:
                    out.setdefault(self.acc_keys[int(k)][0],
                                   set()).add(table.name)
        self._acc_name_clouds = out
        return out

    def row_bytes(self) -> int:
        """Bytes the scan streams per row and pass (DESIGN.md section 3)."""
        return 3 * 8 + 4 * 2

    # ----------------------------------------------------------------- device
    def handle(self, device: int = 0) -> ctypes.c_void_p:
        """Device copy of the table (skyopt_catalog_create), made on first
        use; one replica per GPU (the catalog is small: replicate, don't
        shard -- SURVEY.md section 8e)."""
        hit = self._handles.get(device)
        if hit is not None:
            return hit
        with self._lock:
            hit = self._handles.get(device)
            if hit is not None:
                return hit
            lib = _native.load()
            c = self.columns
            desc = _native.CatalogDesc()
            desc.n_rows = self.n_rows
            keep = []

            def p(name, dtype):
                arr = c[name]
                if arr is None:
                    return None
                arr = np.ascontiguousarray(arr, dtype=dtype)
                keep.append(arr)
                return arr.ctypes.data

            desc.price = p('price', np.float64)
            desc.spot_price = p('spot_price', np.float64)
            desc.vcpus = p('vcpus', np.float64)
            desc.mem = p('mem', np.float64)
            desc.disk_total = p('disk_total', np.float64)
            desc.acc_key = p('acc_key', np.uint16)
            desc.region_id = p('region_id', np.uint16)
            desc.zone_id = p('zone_id', np.uint16)
            desc.flags = p('flags', np.uint16)
            desc.inst_id = p('inst_id', np.int32)
            desc.n_clouds = len(self.clouds)
            desc.n_inst = len(self.inst_names)
            desc.n_acc_keys = len(self.acc_keys)
            desc.n_regions = int(c['cloud_region_offsets'][-1])
            desc.cloud_row_offsets = p('cloud_row_offsets', np.int32)
            desc.cloud_inst_offsets = p('cloud_inst_offsets', np.int32)
            desc.cloud_region_offsets = p('cloud_region_offsets', np.int32)
            desc.cloud_n_zones = p('cloud_n_zones', np.int32)
            desc.region_is_us = p('region_is_us', np.uint8)
            desc.inst_row_offsets = p('inst_row_offsets', np.int32)
            desc.inst_rows = p('inst_rows', np.int32)
            desc.acc_row_offsets = p('acc_row_offsets', np.int32)
            desc.acc_rows = p('acc_rows', np.int32)
            desc.inst_acc_key = p('inst_acc_key', np.uint16)
            zm = np.ascontiguousarray(c['zone_map'])
            keep.append(zm)
            desc.zone_map = zm.ctypes.data
            handle = ctypes.c_void_p(None)
            _native.check(
                lib.skyopt_catalog_create(ctypes.byref(desc), device,
                                          ctypes.byref(handle)))
            del keep
            self._handles[device] = handle
        return handle

    def set_scan_mode(self, mode: str, device: int = 0) -> None:
        """'auto' | 'tile' | 'queue' | 'queue32' (the round-1 row-scoring
        kernels) | 'fast-noprune' (class-table scan in one fused launch, zone
        map and bound ignored: HBM stress) | 'fast-split' /
        'fast-split-noprune' (class-table scan as separate launches)
        (skyopt_catalog_set_scan_mode)."""
        code = {'auto': 0, 'tile': 1, 'queue': 4, 'queue32': 5,
                'fast-noprune': 7, 'fast-split': 8,
                'fast-split-noprune': 9}[mode]
        _native.check(_native.load().skyopt_catalog_set_scan_mode(
            self.handle(device), code))

    def load_images(self, path: str) -> None:
        """`<path>/<cloud>/images.csv` of every loaded cloud (the reference
        reads them with read_catalog('<cloud>/images.csv'),
        sky/catalog/aws_catalog.py:355-372)."""
        for t in self.clouds:
            csv = os.path.join(path, t.name, 'images.csv')
            if os.path.exists(csv):
                self.images[t.name] = pd.read_csv(csv)
        meta = os.path.join(path, 'common', 'metadata.csv')
        if os.path.exists(meta):
            self.metadata = pd.read_csv(meta)

    def set_accelerator_metadata(self, frame: pd.DataFrame) -> None:
        """GPU / MemoryGB / Manufacturer rows (common/metadata.csv)."""
        self.metadata = frame.reset_index(drop=True)

    def set_images(self, cloud: str, frame: pd.DataFrame) -> None:
        self.images[cloud.lower()] = frame.reset_index(drop=True)

    def register_session(self, session) -> None:
        self._sessions.add(session)

    def unregister_session(self, session) -> None:
        self._sessions.discard(session)

    def close(self) -> None:
        # sessions hold the raw catalog handle: close them first (a later
        # resolve() on them raises 'session is closed' instead of touching
        # freed device memory)
        for session in list(self._sessions):
            session.close()
        for handle in list(self._handles.values()):
            _native.load().skyopt_catalog_destroy(handle)
        self._handles.clear()

    def __del__(self):
        try:
            self.close()
        except Exception:  # pylint: disable=broad-except
            pass
