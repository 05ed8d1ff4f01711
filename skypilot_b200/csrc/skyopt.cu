// skyopt.cu -- host side of libskyopt: catalog upload, workspace management
// and the C-ABI entry points declared in include/skyopt.h.
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo
//        -fmad=false -shared -Xcompiler -fPIC  (see __graft_entry__.build()).
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <new>
#include <queue>
#include <string>
#include <thread>
#include <tuple>
#include <unordered_map>
#include <array>
#include <atomic>
#include <vector>

#include "skyopt.h"
#include "skyopt_kernels.cuh"
#include "skyopt_fast.cuh"
#include "skyopt_step.cuh"

using namespace skyopt;

namespace {

thread_local std::string g_error;

int fail(int code, const char *fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_error = buf;
  return code;
}

#define CU(expr)                                                            \
  do {                                                                      \
    cudaError_t e_ = (expr);                                                \
    if (e_ != cudaSuccess)                                                  \
      return fail(SKYOPT_ECUDA, "%s failed: %s (%s:%d)", #expr,             \
                  cudaGetErrorString(e_), __FILE__, __LINE__);              \
  } while (0)

// NVTX range around a native entry point (shows up in Nsight timelines next
// to the host events of skypilot_b200/utils/timeline.py).
struct NvtxRange {
  explicit NvtxRange(const char *name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
};

inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }
inline int next_pow2(int x) { int p = 1; while (p < x) p <<= 1; return p; }

// skyopt_set_chain_paths, process-wide. Bits 0 and 1 are the chain DP's
// force_full (StepArgs::force_full, solve_kernel).
std::atomic<int> g_chain_paths{0};
int chain_force_full() { return g_chain_paths.load(std::memory_order_relaxed) & (SKYOPT_CHAIN_FULL | SKYOPT_CHAIN_GENERAL); }
// skyopt_set_scan_pieces, process-wide
std::atomic<int> g_scan_pieces{0};

// A grow-only allocation that owns its memory: device memory (`kPinned`
// false), zero-filled whenever it is allocated, or pinned host memory. Its
// capacity is a multiple of `quantum` bytes.
template <bool kPinned>
class Buffer {
 public:
  explicit Buffer(size_t quantum = 256) : quantum_(quantum) {}
  Buffer(Buffer &&o) noexcept { *this = std::move(o); }
  Buffer &operator=(Buffer &&o) noexcept {
    std::swap(p_, o.p_); std::swap(cap_, o.cap_); std::swap(quantum_, o.quantum_);
    return *this;
  }
  ~Buffer() { if (p_) kPinned ? cudaFreeHost(p_) : cudaFree(p_); }

  template <typename T = char> T *get() const { return reinterpret_cast<T *>(p_); }

  // Holds at least `bytes` afterwards. A smaller buffer is replaced by one a
  // quarter larger than asked, after `st` (the stream that uses it) has
  // finished with it.
  int reserve(size_t bytes, cudaStream_t st) {
    if (p_ && bytes <= cap_) return 0;
    if (p_) {
      CU(cudaStreamSynchronize(st));
      *this = Buffer(quantum_);
    }
    const size_t cap = std::max(align_up(bytes + bytes / 4, quantum_), quantum_);
    void *p = nullptr;
    cudaError_t e = kPinned ? cudaMallocHost(&p, cap) : cudaMalloc(&p, cap);
    // result fields a kernel does not write for a given problem (e.g. the
    // chosen candidate of a DAG without a plan) are copied back as zeros
    if (e == cudaSuccess && !kPinned && (e = cudaMemsetAsync(p, 0, cap, st)) != cudaSuccess) cudaFree(p);
    if (e != cudaSuccess)
      return fail(SKYOPT_ECUDA, "allocating %zu bytes: %s", cap, cudaGetErrorString(e));
    p_ = static_cast<char *>(p);
    cap_ = cap;
    return 0;
  }

 private:
  char *p_ = nullptr;
  size_t cap_ = 0, quantum_ = 256;
};
using DeviceBuffer = Buffer<false>;
using HostBuffer = Buffer<true>;

// Private stream, events and buffers of one in-flight call.
struct Ctx {
  cudaStream_t stream = nullptr;
  cudaEvent_t ev[8] = {};
  DeviceBuffer dbuf{1 << 20};  // device workspace: a plan, or a session's device-resident plan
  DeviceBuffer scratch;        // a call's temporaries next to the plan: list tables, listings, candidate tables
  HostBuffer hbuf{1 << 16};    // pinned staging
  DeviceBuffer flush;    // skyopt_optimize_timed's L2 flush
  DeviceBuffer trace;    // SKYOPT_TRACE: device-side timeline
  DeviceBuffer sync;     // step_kernel's barrier counter: monotone, never reset in a launch
  unsigned int sync_total = 0;  // arrivals expected so far (the next launch's barrier target)

  ~Ctx() {
    if (stream) cudaStreamDestroy(stream);
    for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
  }
};

// Bump allocator over one buffer; first pass (base == nullptr) only sizes.
struct Carver {
  char *base; size_t off = 0;
  explicit Carver(char *b) : base(b) {}
  template <typename T> T *take(size_t n) {
    off = align_up(off);
    T *p = base ? reinterpret_cast<T *>(base + off) : nullptr;
    off += n * sizeof(T);
    return p;
  }
};

// Lays arrays out in `buf`: `carve` takes them from a Carver, once to size
// the buffer and once to place them.
template <typename F>
int carve_in(DeviceBuffer &buf, cudaStream_t st, F &&carve) {
  Carver sizing(nullptr);
  carve(sizing);
  if (int rc = buf.reserve(sizing.off, st)) return rc;
  Carver c(buf.get());
  carve(c);
  return 0;
}

}  // namespace

struct SkyoptCatalog {
  int device = 0;
  CatDev dev{};
  // Static tile classes. For every tile size (256 << r rows, r = 0..2) the
  // tiles of a cloud are split into those where default-family rows are
  // common ("dense": requests without accelerators match most of their rows)
  // and the rest; each class has its own flag density, so the dense part of a
  // catalog can be scanned with few queries per block and the sparse part
  // with all of them fused.
  struct TileClass {
    int n_tiles = 0;
    int list0 = -1;  // offset into the device tile list; -1 = the run of
    int tile0 = 0;   //   n_tiles consecutive tiles starting at tile0
    // density[m]: fraction of the class's 128-row chunks whose summary carries
    // every flag bit of m -- how often a query requiring m survives the
    // zone-map test (used to size the scan's query groups)
    std::array<float, 256> density{};
  };
  std::vector<std::array<TileClass, 2>> tile_class[3];  // [r][cloud][0 sparse, 1 dense]
  const int32_t *d_tile_list = nullptr;
  std::vector<void *> allocs;
  int64_t device_bytes = 0;
  std::vector<int32_t> cloud_row_offsets, cloud_inst_offsets, cloud_n_zones,
      cloud_region_offsets;
  std::vector<int32_t> cloud_group_cap;  // max rows of one expand group
  int sort_n = 2, max_regions = 1, max_zones = 1;
  int sm_count = 132;
  int64_t l2_bytes = 50ll << 20;
  int scan_mode = 0;  // as set by skyopt_catalog_set_scan_mode: 0, 1, 4, 5, 7, 8 or 9
  // round-2 fast path (skyopt_fast.cuh): rank / class layouts and static
  // launchable orders; fast_ok = the class dictionaries fit shared memory
  FastCat fast{};
  bool fast_ok = false;
  bool coop = false;      // device supports cooperative launches
  std::vector<int32_t> n_cm, n_fa, n_rz;   // class counts per cloud
  std::vector<int32_t> cm_off, fa_off, rz_off;  // [n_clouds + 1] into the dictionaries
  // host copy of the zone map's flags, fixed-host groups and accelerator
  // signature, one array each (the scan planner's cost)
  std::vector<uint32_t> zm_flags, zm_grp, zm_sig_lo, zm_sig_hi;
  int64_t fast_bytes = 0;
  std::mutex mu;
  std::vector<Ctx *> free_ctx;
};

namespace {

template <typename T>
int upload(SkyoptCatalog *c, const T *src, size_t n, size_t slack, const T **dst,
           int fill = 0) {
  T *p = nullptr;
  const size_t bytes = (n + slack) * sizeof(T);
  CU(cudaMalloc(&p, std::max<size_t>(bytes, 256)));
  c->allocs.push_back(p);
  c->device_bytes += bytes;
  CU(cudaMemset(p, fill, std::max<size_t>(bytes, 256)));
  if (n && src) CU(cudaMemcpy(p, src, n * sizeof(T), cudaMemcpyHostToDevice));
  *dst = p;
  return 0;
}

#include "skyopt_fast_host.inc"

// A call's hold on one of the catalog's pooled contexts, from open() (which
// selects the catalog's device and takes a context, or makes one) to its
// destruction. A call that did not end through finish(0) may have left work
// on the stream: it is waited for before the context goes back to the pool.
class Lease {
 public:
  Lease() = default;
  Lease(const Lease &) = delete;
  Lease &operator=(const Lease &) = delete;
  ~Lease() {
    if (!x_) return;
    if (!ok_) cudaStreamSynchronize(x_->stream);
    std::lock_guard<std::mutex> g(cat_->mu);
    cat_->free_ctx.push_back(x_);
  }
  int open(SkyoptCatalog *cat) {
    CU(cudaSetDevice(cat->device));
    cat_ = cat;
    {
      std::lock_guard<std::mutex> g(cat->mu);
      if (!cat->free_ctx.empty()) {
        x_ = cat->free_ctx.back();
        cat->free_ctx.pop_back();
        return 0;
      }
    }
    std::unique_ptr<Ctx> x(new (std::nothrow) Ctx());
    if (!x) return fail(SKYOPT_ENOMEM, "out of host memory");
    CU(cudaStreamCreateWithFlags(&x->stream, cudaStreamNonBlocking));
    for (auto &e : x->ev) CU(cudaEventCreate(&e));
    if (int rc = x->sync.reserve(sizeof(unsigned int), x->stream)) return rc;
    x_ = x.release();
    return 0;
  }
  // The call's result; 0 marks it as succeeded.
  int finish(int rc) { ok_ = rc == 0; return rc; }
  SkyoptCatalog *cat() const { return cat_; }
  Ctx *ctx() const { return x_; }
  Ctx *operator->() const { return x_; }

 private:
  SkyoptCatalog *cat_ = nullptr;
  Ctx *x_ = nullptr;
  bool ok_ = false;
};

// Which kernels a call runs; the values are SkyoptStats::scan_form. The
// row-major scan runs one tile per block or in queue form, followed by expand,
// gather and solve. The class-table scan, placement and chain DP run as
// separate launches or fused into one cooperative step_kernel launch.
enum class Path : int32_t { kTile = 0, kQueue = 2, kSplit = 3, kFused = 4 };

// What one run of a plan launched, as SkyoptStats reports it, and the events
// of Ctx::ev that bracket each of its phases ({0, 0}: not timed).
struct Launched {
  struct Span { int begin = 0, end = 0; };
  Path form = Path::kTile;
  int scan_launches = 0, total_launches = 0, scan_blocks = 0;
  int64_t scan_rows = 0, pass_rows = 0, layout_rows = 0;
  Span scan, expand, solve, scan_kernel;
};

// Everything one call needs, laid out twice (host staging / device).
struct Plan {
  Path path = Path::kTile;
  bool solve = true;      // expand / place and solve follow the scan
  bool finalize = false;  // the caller reads the scan's per-query results
  bool class_tables() const { return path == Path::kSplit || path == Path::kFused; }
  Launched ran;           // what the last enqueue launched
  // sizes
  int nq = 0, nsets = 0, ns = 0, nt = 0, np = 0, ntar = 0, nb = 0, nd = 0, nr = 0, nrb = 1;
  int n_groups = 0, n_blocks = 0, rpt = 4, nsq = 0;
  int64_t n_partials = 0, list_entries = 0, fuzzy_entries = 0;
  int64_t cand_cap = 0;   // expand candidate buffers
  int64_t scan_rows = 0, pass_rows = 0;
  // round-2 fast path (scan2_kernel + place_kernel)
  bool noprune = false; bool fresh_inputs = true; int parity = 0; int n_groups2 = 0, n_pieces = 0, scan2_grid = 0;
  size_t scan2_smem = 0; int64_t layout_rows = 0;
  std::vector<int32_t> piece_chunk0;  // [n_pieces] first chunk of each piece (Scan2Args::inline_chunk0)
  Scan2Group *groups2; const Scan2Group *host_groups2 = nullptr; uint32_t *best_rank, *any_in;
  PlaceTask *ptasks; SlotAux *saux; uint32_t cap_fa = 0, cap_cm = 0, cap_rz = 0;
  int32_t *dag_done; TaskMin *task_mv; uint32_t *shared_tables; unsigned int *group_ready; bool chain_dags = false; bool chain_blocks = false; int step_grid = 0; size_t step_smem = 0;
  // input region (mirrored host/device)
  size_t in_bytes = 0;
  SkyoptQuery *queries; uint32_t *acc_sets; SkyoptSlot *slots; SkyoptTask *tasks;
  int32_t *parents; double *tariffs; SkyoptBlocked *blocked; SkyoptDag *dags;
  SkyoptReservation *resv; int32_t *resv_off;
  ScanQuery *squeries; QueryTest *qtests; ScanGroup *groups; const ScanGroup *host_groups = nullptr; int32_t *partial_base, *partial_count;
  int64_t *list_base, *fuzzy_base, *slot_off, *task_off; int32_t *task_dag;
  // device-only scratch
  ScanPartial *partials; unsigned long long *list_min, *fuzzy_min, *gbest;
  int32_t *cand_region, *cand_zone; double *cand_pa, *cand_pb;
  int32_t *tc_ref, *tc_slot, *tc_cloud; double *tc_hourly, *tc_value, *dp;
  int32_t *back; int32_t *err_flag;
  // output region (device, copied back in one piece)
  size_t out_off = 0, out_bytes = 0;
  ScanFinal *finals; uint32_t *any1; int32_t *slot_count, *slot_inst;
  SkyoptCandidate *chosen; int32_t *chosen_index, *task_n; SkyoptDagResult *dagres;
  int32_t *err_out;
  size_t total_bytes = 0;
};

void carve_inputs(Plan &P, Carver &c) {
  P.queries = c.take<SkyoptQuery>(P.nq);
  P.acc_sets = c.take<uint32_t>((size_t)P.nsets * SKYOPT_ACC_SET_WORDS);
  P.slots = c.take<SkyoptSlot>(P.ns);
  P.tasks = c.take<SkyoptTask>(P.nt);
  P.parents = c.take<int32_t>(P.np);
  P.tariffs = c.take<double>(P.ntar);
  P.blocked = c.take<SkyoptBlocked>(P.nb);
  P.dags = c.take<SkyoptDag>(P.nd);
  P.resv = c.take<SkyoptReservation>(P.nr);
  P.resv_off = c.take<int32_t>(P.nrb + 1);
  P.squeries = c.take<ScanQuery>(P.nsq);
  P.qtests = c.take<QueryTest>(P.nsq);
  P.groups = c.take<ScanGroup>(P.n_groups);
  P.partial_base = c.take<int32_t>(P.nq);
  P.partial_count = c.take<int32_t>(P.nq);
  P.list_base = c.take<int64_t>(P.nq);
  P.fuzzy_base = c.take<int64_t>(P.nq);
  P.slot_off = c.take<int64_t>(P.ns);
  P.task_off = c.take<int64_t>(P.nt + 1);
  P.task_dag = c.take<int32_t>(P.nt);
  P.groups2 = c.take<Scan2Group>(P.n_groups2);
  const bool tables = P.class_tables();
  P.ptasks = c.take<PlaceTask>(tables ? P.nt : 0);
  P.saux = c.take<SlotAux>(tables ? P.ns : 0);
  P.dag_done = c.take<int32_t>(tables ? P.nd : 0);
  // two copies: a launch works on one and re-arms the other for the next
  // launch of a device-resident loop (skyopt_optimize_timed), off its own path
  P.group_ready = c.take<unsigned int>(2 * (size_t)P.n_groups2);
  P.best_rank = c.take<uint32_t>(tables ? 2 * (size_t)P.nq : 0);
  P.any_in = c.take<uint32_t>(tables ? 2 * (size_t)P.nq : 0);
}

// The output region, in the order it is laid out on the device and in the
// pinned buffer it is copied back to.
void carve_outputs(Plan &P, Carver &c) {
  P.finals = c.take<ScanFinal>(P.nq);
  P.any1 = c.take<uint32_t>(P.nq);
  P.slot_count = c.take<int32_t>(P.ns);
  P.slot_inst = c.take<int32_t>(P.ns);
  P.chosen = c.take<SkyoptCandidate>(P.nt);
  P.chosen_index = c.take<int32_t>(P.nt);
  P.task_n = c.take<int32_t>(P.nt);
  P.dagres = c.take<SkyoptDagResult>(P.nd);
  P.err_out = c.take<int32_t>(1);
}

void carve_rest(Plan &P, Carver &c) {
  P.partials = c.take<ScanPartial>(P.n_partials);
  P.list_min = c.take<unsigned long long>(P.list_entries);
  P.fuzzy_min = c.take<unsigned long long>(P.fuzzy_entries);
  P.gbest = c.take<unsigned long long>(P.nsq);
  P.task_mv = c.take<TaskMin>((size_t)P.nt * SKYOPT_MAX_CLOUDS);
  P.shared_tables = c.take<uint32_t>((size_t)P.n_groups2 * (2 * P.cap_fa + P.cap_cm + P.cap_rz));
  P.cand_region = c.take<int32_t>(P.cand_cap);
  P.cand_zone = c.take<int32_t>(P.cand_cap);
  P.cand_pa = c.take<double>(P.cand_cap);
  P.cand_pb = c.take<double>(P.cand_cap);
  P.tc_ref = c.take<int32_t>(P.cand_cap);
  P.tc_slot = c.take<int32_t>(P.cand_cap);
  P.tc_cloud = c.take<int32_t>(P.cand_cap);
  P.tc_hourly = c.take<double>(P.cand_cap);
  P.tc_value = c.take<double>(P.cand_cap);
  P.dp = c.take<double>(P.cand_cap);
  P.back = c.take<int32_t>(P.cand_cap);
  P.err_flag = c.take<int32_t>(1);
  c.off = align_up(c.off);
  P.out_off = c.off;
  carve_outputs(P, c);
  c.off = align_up(c.off);
  P.out_bytes = c.off - P.out_off;
}

// What the expand, place, gather, solve and table kernels see of a plan's
// device buffers.
struct SolveViews {
  ExpandOut ex;
  SolveIn in;
  SolveWork w;
  SolveOut out;
};

SolveViews solve_views(const Plan &P, unsigned long long *trace = nullptr) {
  const ExpandOut ex{P.slot_count, P.slot_inst, P.cand_region, P.cand_zone, P.cand_pa, P.cand_pb};
  return SolveViews{
      ex,
      SolveIn{P.slots, P.tasks, P.parents, P.tariffs, P.blocked, P.dags, P.slot_off, P.task_off, ex, 0, P.resv, P.resv_off},
      SolveWork{P.tc_ref, P.tc_slot, P.tc_cloud, P.tc_hourly, P.tc_value, P.dp, P.back},
      SolveOut{P.chosen, P.chosen_index, P.task_n, P.dagres, trace}};
}

// A reservation table `resv[n]` and its blocks `rr[nrr + 1]` (NULL: one
// block, the whole table): ranges monotone and inside the table, valid keys,
// each block sorted by (cloud, instance type, zone) with unique keys.
int validate_reservations(const SkyoptCatalog *cat, const SkyoptReservation *resv, int n,
                          const int32_t *rr, int nrr) {
  const int C = cat->dev.n_clouds;
  if (n < 0 || (n > 0 && !resv))
    return fail(SKYOPT_EINVAL, "bad reservation table");
  const int n_blocks = rr ? nrr : 1;
  if (rr) {
    if (n_blocks < 0) return fail(SKYOPT_EINVAL, "bad reservation range count %d", n_blocks);
    for (int k = 0; k <= n_blocks; ++k)
      if (rr[k] < 0 || rr[k] > n || (k > 0 && rr[k] < rr[k - 1]))
        return fail(SKYOPT_EINVAL, "reservation range %d: not monotone or outside the table", k);
  }
  for (int i = 0; i < n; ++i) {
    const SkyoptReservation &r = resv[i];
    if (r.cloud < 0 || r.cloud >= C || r.inst_id < 0 || r.inst_id >= cat->dev.n_inst || r.zone_id < 0)
      return fail(SKYOPT_EINVAL, "reservation %d: bad cloud, instance type or zone", i);
  }
  for (int k = 0; k < n_blocks; ++k) {
    const int b = rr ? rr[k] : 0, e = rr ? rr[k + 1] : n;
    for (int i = b + 1; i < e; ++i) {
      const SkyoptReservation &q = resv[i - 1], &r = resv[i];
      if (std::make_tuple(q.cloud, q.inst_id, q.zone_id) >= std::make_tuple(r.cloud, r.inst_id, r.zone_id))
        return fail(SKYOPT_EINVAL, "reservation %d: block %d not sorted by (cloud, instance type, zone) or a key twice", i, k);
    }
  }
  return 0;
}

// `rr` / `nrr`: the reservation blocks (NULL: one block, the whole table).
int validate_problem(const SkyoptCatalog *cat, const SkyoptProblem *pb,
                     const int32_t *rr = nullptr, int nrr = 0) {
  const int C = cat->dev.n_clouds;
  for (int i = 0; i < pb->n_queries; ++i) {
    const SkyoptQuery &q = pb->queries[i];
    if (q.cloud < 0 || q.cloud >= C) return fail(SKYOPT_EINVAL, "query %d: bad cloud %d", i, q.cloud);
    if (q.acc_set >= pb->n_acc_sets || q.fuzzy_set >= pb->n_acc_sets)
      return fail(SKYOPT_EINVAL, "query %d: accelerator set out of range", i);
    if ((q.qflags & SKYOPT_Q_ACC) && q.acc_set < 0)
      return fail(SKYOPT_EINVAL, "query %d: accelerator query without a set", i);
    if (q.price_col != 0 && q.price_col != 1) return fail(SKYOPT_EINVAL, "query %d: bad price_col", i);
  }
  for (int i = 0; i < pb->n_slots; ++i) {
    const SkyoptSlot &s = pb->slots[i];
    if (s.cloud < 0 || s.cloud >= C) return fail(SKYOPT_EINVAL, "slot %d: bad cloud", i);
    if (s.query >= pb->n_queries || s.gate_query >= pb->n_queries)
      return fail(SKYOPT_EINVAL, "slot %d: query out of range", i);
    if (s.query < 0 && s.inst_id < -2) return fail(SKYOPT_EINVAL, "slot %d: no instance type", i);
    if (s.inst_id >= cat->dev.n_inst) return fail(SKYOPT_EINVAL, "slot %d: instance id out of range", i);
    if (s.acc_set >= pb->n_acc_sets) return fail(SKYOPT_EINVAL, "slot %d: accelerator set out of range", i);
    if (s.region_set >= pb->n_acc_sets) return fail(SKYOPT_EINVAL, "slot %d: region set out of range", i);
    if (s.query < 0 && s.inst_id == -1) return fail(SKYOPT_EINVAL, "slot %d: neither query nor instance", i);
  }
  for (int i = 0; i < pb->n_tasks; ++i) {
    const SkyoptTask &t = pb->tasks[i];
    if (t.slot_begin < 0 || t.slot_end < t.slot_begin || t.slot_end > pb->n_slots)
      return fail(SKYOPT_EINVAL, "task %d: bad slot range", i);
    if (t.n_parents < 0 || t.parent_begin < 0 || t.parent_begin + t.n_parents > pb->n_parents)
      return fail(SKYOPT_EINVAL, "task %d: bad parent range", i);
    if (t.n_parents > 0 && (t.edge_tariff_begin < 0 ||
                            t.edge_tariff_begin + t.n_parents * C > pb->n_tariffs))
      return fail(SKYOPT_EINVAL, "task %d: bad tariff range", i);
    if (t.src_tariff_begin >= 0 && t.src_tariff_begin + C > pb->n_tariffs)
      return fail(SKYOPT_EINVAL, "task %d: bad source tariff range", i);
  }
  const int rc = validate_reservations(cat, pb->reservations, pb->n_reservations, rr, nrr);
  if (rc) return rc;
  // the table's blocks: one per context, or the whole table
  const int n_blocks = rr ? nrr : 1;
  for (int i = 0; i < pb->n_slots; ++i)
    if (pb->slots[i].pad_ < 0 || pb->slots[i].pad_ > n_blocks)
      return fail(SKYOPT_EINVAL, "slot %d: reservation block %d out of range", i, pb->slots[i].pad_ - 1);
  for (int i = 0; i < pb->n_dags; ++i) {
    const SkyoptDag &d = pb->dags[i];
    if (d.task_begin < 0 || d.task_end <= d.task_begin || d.task_end > pb->n_tasks)
      return fail(SKYOPT_EINVAL, "dag %d: bad task range", i);
    if (d.blocked_begin < 0 || d.blocked_end < d.blocked_begin || d.blocked_end > pb->n_blocked)
      return fail(SKYOPT_EINVAL, "dag %d: bad blocked range", i);
    if (d.is_chain < SKYOPT_DAG_GENERAL || d.is_chain > SKYOPT_DAG_SAME_INFRA)
      return fail(SKYOPT_EINVAL, "dag %d: unknown kind %d", i, d.is_chain);
    const bool chain = d.is_chain == SKYOPT_DAG_CHAIN;
    for (int t = d.task_begin; t < d.task_end; ++t) {
      const SkyoptTask &tk = pb->tasks[t];
      for (int k = 0; k < tk.n_parents; ++k) {
        const int lp = pb->parents[tk.parent_begin + k];
        if (lp < 0 || lp >= t - d.task_begin)
          return fail(SKYOPT_EINVAL, "dag %d: task order is not topological", i);
      }
      if (chain && tk.n_parents != (t == d.task_begin ? 0 : 1))
        return fail(SKYOPT_EINVAL, "dag %d: not a chain", i);
      if (chain && tk.n_parents == 1 && pb->parents[tk.parent_begin] != t - d.task_begin - 1)
        return fail(SKYOPT_EINVAL, "dag %d: chain parent must be the previous task", i);
      if (d.is_chain == SKYOPT_DAG_SAME_INFRA && tk.n_parents != 0)
        return fail(SKYOPT_EINVAL, "dag %d: a job group's task %d has parents", i, t - d.task_begin);
    }
  }
  return 0;
}

// The class-table path takes plain argmin queries (no list / fuzzy tables),
// single-key accelerator slots and tasks of at most kFastMaxTaskSlots slots,
// on catalogs whose class dictionaries fit shared memory.
bool takes_class_tables(const SkyoptCatalog *cat, const SkyoptProblem *pb) {
  if (!cat->fast_ok || !(cat->scan_mode == 0 || cat->scan_mode >= 7)) return false;
  for (int i = 0; i < pb->n_queries; ++i)
    if (pb->queries[i].qflags & (SKYOPT_Q_LIST | SKYOPT_Q_FUZZY)) return false;
  for (int s = 0; s < pb->n_slots; ++s) {
    const int set = pb->slots[s].acc_set;
    if (set < 0) continue;
    int bits = 0;
    const uint32_t *w = pb->acc_sets + (size_t)set * SKYOPT_ACC_SET_WORDS;
    for (int k = 0; k < SKYOPT_ACC_SET_WORDS; ++k) bits += __builtin_popcount(w[k]);
    if (bits > 1) return false;  // several spellings of one accelerator: merge needs a sort
  }
  for (int t = 0; t < pb->n_tasks; ++t)
    if (pb->tasks[t].slot_end - pb->tasks[t].slot_begin > kFastMaxTaskSlots) return false;
  return true;
}

// The weighted piece plan's estimate of a scan block's time, in ns: per
// mask-table entry of its slice, per chunk it tests against the zone map and
// per chunk it scores. kCostVisit and kCostLive are fitted to SKYOPT_TRACE
// timelines of the cfg4 fused step on an H100; kCostEntry is the table
// build's own work, which those timelines cannot resolve (DESIGN §4). Only
// the ratios matter.
constexpr double kCostEntry = 5.0, kCostVisit = 23.0, kCostLive = 68.0;

// Class-table scan: groups of <= 32 queries per (cloud, price column), cut
// into pieces of consecutive 128-row chunks for a grid that is resident at
// once, and where the fused step runs each DAG's chain DP. The grid is sized
// for the kernel that P.path launches. `order2`: scan order -> the caller's
// query index.
void group_class_tables(const SkyoptCatalog *cat, const SkyoptProblem *pb,
                        const std::vector<std::vector<int>> &by_cloud, Plan &P,
                        std::vector<Scan2Group> &groups2, std::vector<int> &order2) {
  const int C = cat->dev.n_clouds;
  std::vector<char> gate_used(std::max(P.nq, 1), 0);
  for (int sl = 0; sl < P.ns; ++sl) if (pb->slots[sl].gate_query >= 0) gate_used[pb->slots[sl].gate_query] = 1;
  long long visits = 0;
  for (int c = 0; c < C; ++c)
    for (int col = 0; col < 2; ++col) {
      std::vector<int> qs;
      for (int qi : by_cloud[c]) if ((pb->queries[qi].price_col ? 1 : 0) == col) qs.push_back(qi);
      for (size_t b = 0; b < qs.size(); b += kQChunk) {
        Scan2Group G{};
        G.cloud = c; G.col = col; G.q_begin = (int)order2.size();
        G.q_count = (int)std::min<size_t>(kQChunk, qs.size() - b);
        G.n_cm = cat->n_cm[c]; G.n_fa = cat->n_fa[c]; G.n_rz = cat->n_rz[c];
        G.cm_off = cat->cm_off[c]; G.fa_off = cat->fa_off[c]; G.rz_off = cat->rz_off[c];
        G.chunk0 = cat->cloud_row_offsets[c] / kZoneRows;
        G.n_chunks = cat->cloud_row_offsets[c + 1] / kZoneRows - G.chunk0;
        for (int k = 0; k < G.q_count; ++k) { order2.push_back(qs[b + k]); if (gate_used[qs[b + k]]) G.need_any = 1; }
        if (P.ns == 0) G.need_any = 1;  // skyopt_scan: every result carries any_stage1
        if (G.n_chunks > 0) groups2.push_back(G);
        visits += G.n_chunks;
        P.cap_fa = std::max(P.cap_fa, (uint32_t)G.n_fa); P.cap_cm = std::max(P.cap_cm, (uint32_t)G.n_cm);
        P.cap_rz = std::max(P.cap_rz, (uint32_t)G.n_rz);
      }
    }
  P.cap_fa = (P.cap_fa + 3u) & ~3u; P.cap_cm = (P.cap_cm + 3u) & ~3u; P.cap_rz = (P.cap_rz + 3u) & ~3u;
  P.scan2_smem = scan2_smem_bytes(P.cap_fa, P.cap_cm, P.cap_rz);
  P.step_smem = std::max(P.scan2_smem, std::max(sizeof(PlaceSmem), sizeof(ChainSmem))) + 16;
  int per_sm = kScanBlocksPerSM;
  {
    static std::mutex occ_mu;
    std::lock_guard<std::mutex> g(occ_mu);
    // the separate-launch scan (4 blocks of 61 registers per SM) has more
    // resident blocks than the fused kernel (3)
    const cudaError_t oe = P.path == Path::kFused
        ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, step_kernel, kScanThreads, P.step_smem)
        : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, scan2_kernel, kScanThreads, P.scan2_smem);
    if (oe != cudaSuccess || per_sm < 1) per_sm = 1;
  }
  const long long resident = (long long)per_sm * cat->sm_count;
  // Pieces of consecutive chunks: at most one per resident block (a second
  // piece of another group would re-stage and rebuild the tables), at most
  // one per kMinPiece chunks of the group.
  constexpr long long kMinPiece = 8;
  const long long spare = std::max<long long>(0, resident - (long long)groups2.size());
  const bool weighted = !P.noprune && spare > 0 && resident <= kInlinePieces &&
                        !(g_scan_pieces.load(std::memory_order_relaxed) & SKYOPT_SCAN_PIECES_EQUAL);
  // weighted: per group, how many of its first j chunks pass (j = 0..n_chunks)
  std::vector<std::vector<int32_t>> live;
  auto chunk_cost = [&](size_t g, int j) { return kCostVisit * j + kCostLive * live[g][j]; };
  if (weighted) {
    // A block's time is about c_e per mask-table entry of its slice, c_v per
    // chunk it tests and c_l per chunk it scores (DESIGN §4). The host cannot
    // know the bound, so a chunk counts as scored when it passes the zone-map
    // test for some query of the group. Queries of one (flags, fixed-host
    // group) share a test: a chunk passes some accelerator query of them iff
    // it passes the union of their signatures.
    std::vector<long long> k(groups2.size(), 1), kmax(groups2.size());
    std::vector<double> total(groups2.size());
    std::vector<uint8_t> pass;
    live.resize(groups2.size());
    for (size_t g = 0; g < groups2.size(); ++g) {
      const Scan2Group &G = groups2[g];
      std::vector<std::array<uint32_t, 5>> tests;  // req, grp, accelerator queries, sig_lo, sig_hi
      for (int i = 0; i < G.q_count; ++i) {
        const SkyoptQuery &q = pb->queries[order2[G.q_begin + i]];
        const QueryS s = make_query_s(q);
        const uint32_t acc = (q.qflags & SKYOPT_Q_ACC) ? 1u : 0u;
        uint32_t lo = 0, hi = 0;
        if (acc) {  // as fill_record: no fuzzy sets on this path
          const uint32_t *w = pb->acc_sets + (size_t)q.acc_set * SKYOPT_ACC_SET_WORDS;
          for (int x = 0; x < SKYOPT_ACC_SET_WORDS; ++x) (x & 1 ? hi : lo) |= w[x];
        }
        auto t = std::find_if(tests.begin(), tests.end(), [&](const std::array<uint32_t, 5> &u) {
          return u[0] == s.req_flags && u[1] == s.grp_bit && u[2] == acc;
        });
        if (t == tests.end()) tests.push_back({s.req_flags, s.grp_bit, acc, lo, hi});
        else { (*t)[3] |= lo; (*t)[4] |= hi; }
      }
      const uint32_t *fl = cat->zm_flags.data() + G.chunk0, *gr = cat->zm_grp.data() + G.chunk0;
      const uint32_t *lo = cat->zm_sig_lo.data() + G.chunk0, *hi = cat->zm_sig_hi.data() + G.chunk0;
      pass.assign(G.n_chunks, 0);
      for (const auto &t : tests)  // (branch-free: the compiler vectorises it)
        for (int c = 0; c < G.n_chunks; ++c)
          pass[c] |= (uint8_t)(((fl[c] & t[0]) == t[0]) & ((gr[c] & t[1]) == t[1]) &
                               ((t[2] == 0u) | (((t[3] & lo[c]) | (t[4] & hi[c])) != 0u)));
      std::vector<int32_t> &L = live[g];
      L.assign(G.n_chunks + 1, 0);
      for (int c = 0; c < G.n_chunks; ++c) L[c + 1] = L[c] + pass[c];
      total[g] = (double)(G.n_fa + G.n_cm + G.n_rz) * kCostEntry + chunk_cost(g, G.n_chunks);
      kmax[g] = std::max<long long>(1, G.n_chunks / kMinPiece);
    }
    // the spare blocks one at a time to the group whose blocks cost the most
    std::priority_queue<std::pair<double, size_t>> heap;
    for (size_t g = 0; g < groups2.size(); ++g)
      if (k[g] < kmax[g]) heap.push({total[g], g});
    for (long long left = spare; left > 0 && !heap.empty(); --left) {
      const size_t g = heap.top().second;
      heap.pop();
      if (++k[g] < kmax[g]) heap.push({total[g] / (double)k[g], g});
    }
    for (size_t g = 0; g < groups2.size(); ++g) groups2[g].n_pieces = (int)k[g];
  }
  int piece0 = 0;
  P.piece_chunk0.clear();
  for (Scan2Group &G : groups2) {
    const size_t g = &G - groups2.data();
    if (!weighted) {
      long long k = 1 + (visits > 0 ? spare * G.n_chunks / visits : 0);
      k = std::min<long long>(k, std::max<long long>(1, G.n_chunks / kMinPiece));
      G.n_pieces = (int)std::max<long long>(1, std::min<long long>(k, G.n_chunks));
    }
    G.piece0 = piece0; G.index = (int)g;
    for (int pi = 0; pi < G.n_pieces; ++pi) {
      int b = (int)((int64_t)G.n_chunks * pi / G.n_pieces);  // equal chunk counts
      if (weighted && pi > 0) {
        // the first chunk where the prefix reaches pi / n_pieces of the cost,
        // leaving every piece at least one chunk
        const double want = chunk_cost(g, G.n_chunks) * pi / G.n_pieces;
        int lo = 0, hi = G.n_chunks;
        while (lo < hi) {
          const int mid = (lo + hi) / 2;
          if (chunk_cost(g, mid) < want) lo = mid + 1; else hi = mid;
        }
        b = std::max(lo, P.piece_chunk0.back() - G.chunk0 + 1);
        b = std::min(b, G.n_chunks - (G.n_pieces - pi));
      }
      P.piece_chunk0.push_back(G.chunk0 + b);
    }
    piece0 += G.n_pieces;
    P.layout_rows += (long long)G.n_chunks * kZoneRows;
  }
  P.n_groups2 = (int)groups2.size(); P.n_pieces = piece0;
  P.scan2_grid = (int)std::min<long long>(resident, std::max(P.n_pieces, 1));
  P.chain_dags = true;
  for (int d = 0; d < P.nd; ++d)
    if (pb->dags[d].is_chain != SKYOPT_DAG_CHAIN || pb->dags[d].task_end - pb->dags[d].task_begin > kFastTasks) P.chain_dags = false;
  // Each DAG's chain DP on a block of its own, started from the minima as
  // the task blocks publish them, when the grid holds one block per task and
  // per DAG; else (e.g. thousands of one-task DAGs) on the block that places
  // the DAG's last task. SKYOPT_CHAIN_LAST_TASK_BLOCK (tests) forces the latter.
  P.chain_blocks = P.chain_dags && P.nd > 0 && !(g_chain_paths.load(std::memory_order_relaxed) & SKYOPT_CHAIN_LAST_TASK_BLOCK) &&
                   (long long)P.nt + P.nd <= resident;
  P.step_grid = (int)std::min<long long>(resident, std::max<long long>(piece0, P.chain_blocks ? (long long)P.nt + P.nd : P.nt));
  P.nsq = (int)order2.size();
}

// A unit of the row-major scan: a (cloud, tile class) pair with its own query
// groups. n_tiles: tiles of the unit; n_blocks: blocks of each of its groups;
// tpb: tiles per block (strided over the unit's tile list); cuts: group
// boundaries in the cloud's query list.
struct Unit { int cloud, n_tiles, n_blocks, tpb, list0, tile0; std::vector<int> cuts; };

// The units for tiles of 256 * rpt rows; returns the blocks they launch. Up
// to 32 queries share one pass over a unit's rows. A row chunk that many
// queries match at once is scored query by query by one warp, so groups are
// cut early when the expected number of queries surviving the zone-map test
// per chunk (the class's flag density; accelerator and fixed-host queries are
// selective by key) reaches kDenseCut: the dense tiles of the catalog are then
// spread over more blocks instead of forming the tail of the launch, while
// the sparse tiles keep all queries fused. target_pairs > 0: queue form.
long long make_units(const SkyoptCatalog *cat, const SkyoptProblem *pb,
                     const std::vector<std::vector<int>> &by_cloud, int rpt,
                     std::vector<Unit> &units, float target_pairs = 0.f) {
  constexpr float kDenseCut = 3.0f;
  long long blocks = 0;
  units.clear();
  const int tile = kScanThreads * rpt;
  const int r = rpt == 4 ? 2 : (rpt == 2 ? 1 : 0);
  for (int c = 0; c < cat->dev.n_clouds; ++c) {
    const auto &qs = by_cloud[c];
    if (qs.empty()) continue;
    for (int k = 0; k < 2; ++k) {
      const SkyoptCatalog::TileClass &tc = cat->tile_class[r][c][k];
      if (tc.n_tiles == 0) continue;
      Unit u; u.cloud = c; u.tpb = 1;
      u.n_tiles = tc.n_tiles; u.list0 = tc.list0; u.tile0 = tc.tile0;
      const float *density = tc.density.data();
      u.cuts.push_back(0);
      float dens = 0.f, dmax = 0.f; int n = 0;
      for (size_t i = 0; i < qs.size(); ++i) {
        const SkyoptQuery &q = pb->queries[qs[i]];
        float dq = density[(q.flags_require | SKYOPT_F_VALID) & 0xFFu];
        if ((q.qflags & SKYOPT_Q_ACC) || q.group != 0) dq *= 0.05f;
        if (n > 0 && (n == kQChunk || dens + dq > kDenseCut)) {
          u.cuts.push_back((int)i); dens = 0.f; n = 0;
        }
        dens += dq; ++n;
        dmax = std::max(dmax, dens);
      }
      u.cuts.push_back((int)qs.size());
      if (target_pairs > 0.f) {
        // queue form: as many tiles per block (at most 32: one tested chunk
        // per thread) as keep the expected number of surviving (chunk,
        // query) pairs of the unit's densest group near the target
        const float per_tile = (float)(tile / 128) * std::max(dmax, 1e-3f);
        u.tpb = std::min(32, std::max(1, (int)(target_pairs / per_tile)));
      }
      u.n_blocks = (u.n_tiles + u.tpb - 1) / u.tpb;
      blocks += (long long)u.n_blocks * (long long)(u.cuts.size() - 1);
      units.push_back(std::move(u));
    }
  }
  return blocks;
}

// Row-major scan: its units and its form, one tile per block or the queue
// form, and the tile size (256 * rpt rows).
Path group_units(const SkyoptCatalog *cat, const SkyoptProblem *pb,
                 const std::vector<std::vector<int>> &by_cloud, int &rpt, std::vector<Unit> &units) {
  const long long wave = 2ll * cat->sm_count;
  rpt = 4;
  if (cat->scan_mode < 4 && (cat->scan_mode == 1 || make_units(cat, pb, by_cloud, 4, units) < 3 * wave)) {
    // One tile of 256*rpt rows per block (rows go straight to registers),
    // with smaller tiles when there is too little work to cover all SMs.
    if (make_units(cat, pb, by_cloud, 4, units) < wave) {
      rpt = 2;
      if (make_units(cat, pb, by_cloud, 2, units) < wave) { rpt = 1; make_units(cat, pb, by_cloud, 1, units); }
    }
    return Path::kTile;
  }
  // Queue form (scan_queue_kernel): blocks own several tiles and their
  // warps share the surviving (chunk, query) pairs. The target number of
  // pairs per block is the smallest that lets the whole grid be resident
  // at once (kScanBlocksPerSM blocks per SM, a tenth left free): a second
  // wave would start behind blocks that live 8-12 us
  // (measured on the round-1 kernels).
  const long long resident = (long long)(0.9 * kScanBlocksPerSM * cat->sm_count);
  float target = 16.f;
  if (cat->scan_mode == 5) target = 1e9f;  // tests: 32 tiles per block everywhere
  while (make_units(cat, pb, by_cloud, 4, units, target) > resident && target < 256.f)
    target = target < 64.f ? target + 8.f : target * 1.5f;
  return Path::kQueue;
}

// Sizes, scan grouping and offsets; fills the host staging copy. `solve`:
// expand / place and solve follow the scan; `want_scan_results`: the caller
// reads the scan's per-query results. Decides P.path, the kernels the call
// runs.
int build_plan(const SkyoptCatalog *cat, const SkyoptProblem *pb, Ctx *x, bool solve,
               bool want_scan_results, Plan &P, const int32_t *rr = nullptr, int nrr = 0) {
  const int C = cat->dev.n_clouds;
  P.nq = pb->n_queries; P.nsets = pb->n_acc_sets; P.ns = pb->n_slots;
  P.nt = pb->n_tasks; P.np = pb->n_parents; P.ntar = pb->n_tariffs;
  P.nb = pb->n_blocked; P.nd = pb->n_dags; P.nr = pb->n_reservations;
  P.nrb = rr ? nrr : 1;
  P.solve = solve;
  P.finalize = want_scan_results || !solve;
  P.noprune = cat->scan_mode == 7 || cat->scan_mode == 9;

  std::vector<std::vector<int>> by_cloud(C);
  for (int i = 0; i < P.nq; ++i) by_cloud[pb->queries[i].cloud].push_back(i);
  std::vector<Unit> units;
  std::vector<Scan2Group> groups2;
  std::vector<int> order2;
  if (takes_class_tables(cat, pb)) {
    // the whole step in one cooperative launch, unless the caller reads the
    // scan's results, the mode asks for separate launches or the device
    // cannot launch cooperatively
    const bool split = cat->scan_mode == 8 || cat->scan_mode == 9;
    P.path = solve && !want_scan_results && P.nt && cat->coop && !split ? Path::kFused : Path::kSplit;
    group_class_tables(cat, pb, by_cloud, P, groups2, order2);
  } else {
    P.path = group_units(cat, pb, by_cloud, P.rpt, units);
  }
  std::vector<int> cloud_tiles(C, 0);  // partial slots of one query of the cloud
  for (const Unit &u : units) {
    P.n_groups += (int)u.cuts.size() - 1;
    P.nsq += (int)by_cloud[u.cloud].size();
    cloud_tiles[u.cloud] += u.n_blocks;
  }

  // candidate capacity: every slot can at most expand to its cloud's largest
  // instance-type / accelerator group
  std::vector<int64_t> slot_off(P.ns);
  int64_t cap = 0;
  for (int s = 0; s < P.ns; ++s) { slot_off[s] = cap; cap += cat->cloud_group_cap[pb->slots[s].cloud]; }
  P.cand_cap = cap;

  // partial / table offsets
  std::vector<int32_t> pbase(P.nq), pcount(P.nq);
  std::vector<int64_t> lbase(P.nq, 0), fbase(P.nq, 0);
  int64_t npart = 0, nlist = 0, nfuzzy = 0;
  P.scan_rows = 0;
  for (int i = 0; i < P.nq; ++i) {
    const SkyoptQuery &q = pb->queries[i];
    const int rows = cat->cloud_row_offsets[q.cloud + 1] - cat->cloud_row_offsets[q.cloud];
    pcount[i] = cloud_tiles[q.cloud];
    if (npart + pcount[i] > 0x7FFFFFFFll) return fail(SKYOPT_ELIMIT, "too many scan partials");
    pbase[i] = (int32_t)npart; npart += pcount[i];
    P.scan_rows += rows;
    if (q.qflags & SKYOPT_Q_LIST) { lbase[i] = nlist; nlist += cat->cloud_inst_offsets[q.cloud + 1] - cat->cloud_inst_offsets[q.cloud]; }
    if (q.qflags & SKYOPT_Q_FUZZY) { fbase[i] = nfuzzy; nfuzzy += cat->dev.n_acc_keys; }
  }
  P.n_partials = npart; P.list_entries = nlist; P.fuzzy_entries = nfuzzy;

  Carver sizing(nullptr);
  carve_inputs(P, sizing);
  P.in_bytes = align_up(sizing.off);
  carve_rest(P, sizing);
  P.total_bytes = align_up(sizing.off);
  int rc = x->dbuf.reserve(P.total_bytes, x->stream);
  if (rc) return rc;
  if ((rc = x->hbuf.reserve(std::max(P.in_bytes, P.out_bytes), x->stream))) return rc;

  // host staging copy of the input region
  Carver h(x->hbuf.get());
  carve_inputs(P, h);
  memcpy(P.queries, pb->queries, sizeof(SkyoptQuery) * P.nq);
  if (P.nsets) memcpy(P.acc_sets, pb->acc_sets, sizeof(uint32_t) * SKYOPT_ACC_SET_WORDS * P.nsets);
  if (P.ns) memcpy(P.slots, pb->slots, sizeof(SkyoptSlot) * P.ns);
  if (P.nt) memcpy(P.tasks, pb->tasks, sizeof(SkyoptTask) * P.nt);
  if (P.np) memcpy(P.parents, pb->parents, sizeof(int32_t) * P.np);
  if (P.ntar) memcpy(P.tariffs, pb->tariffs, sizeof(double) * P.ntar);
  if (P.nb) memcpy(P.blocked, pb->blocked, sizeof(SkyoptBlocked) * P.nb);
  if (P.nd) memcpy(P.dags, pb->dags, sizeof(SkyoptDag) * P.nd);
  if (P.nr) memcpy(P.resv, pb->reservations, sizeof(SkyoptReservation) * P.nr);
  if (rr) {
    memcpy(P.resv_off, rr, sizeof(int32_t) * (P.nrb + 1));
  } else {
    P.resv_off[0] = 0; P.resv_off[1] = P.nr;
  }
  memcpy(P.partial_base, pbase.data(), sizeof(int32_t) * P.nq);
  memcpy(P.partial_count, pcount.data(), sizeof(int32_t) * P.nq);
  memcpy(P.list_base, lbase.data(), sizeof(int64_t) * P.nq);
  memcpy(P.fuzzy_base, fbase.data(), sizeof(int64_t) * P.nq);
  if (P.ns) memcpy(P.slot_off, slot_off.data(), sizeof(int64_t) * P.ns);
  // task candidate capacity = sum of its slots' capacities
  {
    int64_t off = 0;
    for (int t = 0; t < P.nt; ++t) {
      P.task_off[t] = off;
      for (int s = pb->tasks[t].slot_begin; s < pb->tasks[t].slot_end; ++s)
        off += cat->cloud_group_cap[pb->slots[s].cloud];
    }
    P.task_off[P.nt] = off;
    if (off > P.cand_cap) {
      // slots shared by several tasks would overflow the task arrays
      return fail(SKYOPT_EINVAL, "a slot belongs to more than one task");
    }
  }
  for (int t = 0; t < P.nt; ++t) P.task_dag[t] = 0;
  for (int d = 0; d < P.nd; ++d)
    for (int t = pb->dags[d].task_begin; t < pb->dags[d].task_end; ++t) P.task_dag[t] = d;
  auto fill_record = [&](ScanQuery &R, int qi) {
    const SkyoptQuery &q = pb->queries[qi];
    memset(&R, 0, sizeof(R));
    R.s = make_query_s(q);
    R.qid = qi;
    R.list_base = lbase[qi];
    R.fuzzy_base = fbase[qi];
    uint32_t lo32 = 0, hi32 = 0;
    const int set_idx[2] = {(q.qflags & SKYOPT_Q_ACC) ? q.acc_set : -1,
                            (q.qflags & SKYOPT_Q_FUZZY) ? q.fuzzy_set : -1};
    for (int which = 0; which < 2; ++which) {
      if (set_idx[which] < 0) continue;
      const uint32_t *src = pb->acc_sets + (size_t)set_idx[which] * SKYOPT_ACC_SET_WORDS;
      for (int w = 0; w < SKYOPT_ACC_SET_WORDS; ++w) {
        R.set[which][w] = src[w];
        if (w & 1) hi32 |= src[w]; else lo32 |= src[w];
      }
    }
    // 64-bit signature (key id mod 64) of the keys the query can match
    R.s.sig_lo = (q.qflags & SKYOPT_Q_ACC) ? lo32 : 0xFFFFFFFFu;
    R.s.sig_hi = (q.qflags & SKYOPT_Q_ACC) ? hi32 : 0xFFFFFFFFu;
  };
  if (P.class_tables()) {
    for (int i = 0; i < P.nsq; ++i) fill_record(P.squeries[i], order2[i]);
    memcpy(P.groups2, groups2.data(), sizeof(Scan2Group) * groups2.size());
    memset(P.best_rank, 0xFF, sizeof(uint32_t) * 2 * P.nq);
    memset(P.any_in, 0, sizeof(uint32_t) * 2 * P.nq);
    if (P.nd) memset(P.dag_done, 0, sizeof(int32_t) * P.nd);
    if (P.n_groups2) memset(P.group_ready, 0, sizeof(unsigned int) * 2 * P.n_groups2);
    // what a task block / a slot needs, in one record each
    for (int t = 0; t < P.nt; ++t) {
      const SkyoptDag &D = pb->dags[P.task_dag[t]];
      PlaceTask &T = P.ptasks[t];
      T.slot_begin = pb->tasks[t].slot_begin; T.slot_end = pb->tasks[t].slot_end;
      T.blocked_begin = D.blocked_begin; T.blocked_end = D.blocked_end;
      T.minimize_cost = D.minimize_cost; T.pad_[0] = T.pad_[1] = T.pad_[2] = 0;
    }
    for (int sl = 0; sl < P.ns; ++sl) {
      const SkyoptSlot &S = pb->slots[sl];
      SlotAux &X = P.saux[sl];
      memset(&X, 0, sizeof(X));
      X.max_price = 1.0 / 0.0;
      if (S.query >= 0) {
        const SkyoptQuery &Q = pb->queries[S.query];
        X.rec_base = cat->cloud_row_offsets[Q.cloud]; X.qcol = Q.price_col ? 1 : 0; X.max_price = Q.max_price;
      }
      X.cloud_r0 = cat->cloud_row_offsets[S.cloud]; X.cloud_r1 = cat->cloud_row_offsets[S.cloud + 1];
      X.has_zones = cat->cloud_n_zones[S.cloud] > 0 ? 1 : 0;
      X.acc_list_key = -1;
      if (S.acc_set >= 0) {
        const uint32_t *w = pb->acc_sets + (size_t)S.acc_set * SKYOPT_ACC_SET_WORDS;
        for (int k = 0; k < SKYOPT_ACC_SET_WORDS && X.acc_list_key < 0; ++k)
          if (w[k]) X.acc_list_key = (int16_t)(32 * k + __builtin_ctz(w[k]));
      }
    }
  }
  int g = 0, qpos = 0, block0 = 0;
  P.pass_rows = 0;
  std::vector<int> unit_pbase(C, 0);  // partial slots used by earlier units of the cloud
  for (int c = 0; c < C; ++c) {
    // algorithmic passes: the minimum (32 fused queries per pass over the
    // cloud's rows), whatever grouping is chosen
    const int rows = cat->cloud_row_offsets[c + 1] - cat->cloud_row_offsets[c];
    P.pass_rows += (int64_t)rows * (int64_t)((by_cloud[c].size() + kQChunk - 1) / kQChunk);
  }
  for (const Unit &u : units) {
    const int c = u.cloud;
    const auto &qs = by_cloud[c];
    const int tiles = u.n_blocks;  // blocks of each group of the unit
    for (size_t ci = 0; ci + 1 < u.cuts.size(); ++ci) {
      const size_t b = (size_t)u.cuts[ci];
      const int n = u.cuts[ci + 1] - u.cuts[ci];
      ScanGroup G{};
      G.row_begin = cat->cloud_row_offsets[c];
      G.row_end = cat->cloud_row_offsets[c + 1];
      G.q_begin = qpos; G.q_count = n; G.block0 = block0; G.n_tiles = tiles;
      G.tiles_per_block = u.tpb; G.total_tiles = u.n_tiles;
      G.list0 = u.list0; G.tile0 = u.tile0;
      for (int k = 0; k < n; ++k) {
        const int qi = qs[b + k];
        const SkyoptQuery &q = pb->queries[qi];
        G.need |= q.price_col ? 2u : 1u;
        if (q.qflags & SKYOPT_Q_FUZZY) G.need |= 1u;
        // the staged record: constraint vector, offsets and key bitmasks
        ScanQuery &R = P.squeries[qpos + k];
        fill_record(R, qi);
        R.partial_base = pbase[qi] + unit_pbase[c];
        QueryTest &T = P.qtests[qpos + k];
        T.req_flags = R.s.req_flags; T.grp_bit = R.s.grp_bit;
        T.sig_lo = R.s.sig_lo; T.sig_hi = R.s.sig_hi;
        T.qflags = R.s.qflags; T.price_col = (uint32_t)(R.s.price_col ? 1 : 0);
        T.partial_base = R.partial_base; T.pad_ = 0;
      }
      P.groups[g++] = G;
      qpos += n; block0 += tiles;
    }
    unit_pbase[c] += tiles;
  }
  P.n_blocks = block0;

  const ScanGroup *host_groups = P.groups;
  P.host_groups2 = P.groups2;
  // device views
  Carver d(x->dbuf.get());
  carve_inputs(P, d);
  carve_rest(P, d);
  P.host_groups = host_groups;  // pinned staging copy stays valid for the call
  return 0;
}

// Starts the record of one run of P: the rows its scan covers, nothing
// launched yet.
Launched &new_record(Plan &P, Path form, int scan_blocks) {
  P.ran = Launched{};
  P.ran.form = form;
  P.ran.scan_blocks = scan_blocks;
  P.ran.scan_rows = P.scan_rows; P.ran.pass_rows = P.pass_rows; P.ran.layout_rows = P.layout_rows;
  return P.ran;
}

// Class-table path: step_kernel (+ solve_kernel for DAGs that are not short
// chains), or scan2 -> [finalize2] -> place -> solve. P.fresh_inputs: the
// scan results were just initialised by the H2D copy of the input region;
// later iterations of the device-resident timing loop reset them with one
// memset.
int enqueue_fast(SkyoptCatalog *cat, Ctx *x, Plan &P) {
  cudaStream_t st = x->stream;
  unsigned long long *trace = x->trace.get<unsigned long long>();
  CU(cudaEventRecord(x->ev[1], st));
  Scan2Args sa{};
  sa.cat = cat->dev; sa.f = cat->fast; sa.squeries = P.squeries; sa.groups = P.groups2;
  sa.n_groups = P.n_groups2; sa.n_pieces = P.n_pieces;
  // fused launches alternate between the two copies of the scan results
  const size_t par = (size_t)(P.parity & 1), oth = par ^ 1;
  uint32_t *best_rank = P.best_rank + par * P.nq, *any_in = P.any_in + par * P.nq;
  sa.best_rank = best_rank; sa.any1 = any_in;
  sa.zero_flag = P.err_out; sa.cap_fa = P.cap_fa; sa.cap_cm = P.cap_cm; sa.cap_rz = P.cap_rz;
  sa.trace = trace; sa.shared_tables = nullptr; sa.group_ready = nullptr;
  for (int i = 0; i < std::min(P.n_groups2, kInlineGroups2); ++i) {
    sa.inline_groups[i] = P.host_groups2[i]; sa.inline_piece0[i] = P.host_groups2[i].piece0;
  }
  if (P.n_pieces <= kInlinePieces) std::copy(P.piece_chunk0.begin(), P.piece_chunk0.end(), sa.inline_chunk0);
  sa.noprune = P.noprune ? 1u : 0u;
  sa.force_any = P.finalize ? 1u : 0u;
  const SolveViews v = solve_views(P, trace);
  if (P.path == Path::kFused) {
    // ---- the whole step in one cooperative launch
    StepArgs sp{};
    sp.scan = sa;
    sp.scan.shared_tables = P.shared_tables; sp.scan.group_ready = P.group_ready + par * P.n_groups2;
    sp.next_best_rank = P.best_rank + oth * P.nq; sp.next_any1 = P.any_in + oth * P.nq;
    sp.next_group_ready = P.group_ready + oth * P.n_groups2;
    sp.force_full = chain_force_full();
    sp.place.cat = cat->dev; sp.place.f = cat->fast; sp.place.ptasks = P.ptasks; sp.place.saux = P.saux;
    sp.place.best_rank = best_rank; sp.place.any1 = any_in; sp.place.acc_sets = P.acc_sets;
    sp.place.in = v.in; sp.place.w = v.w; sp.place.task_n = P.task_n; sp.place.trace = trace;
    sp.place.task_mv = P.task_mv;
    sp.out = v.out;
    sp.task_dag = P.task_dag; sp.n_tasks = P.nt; sp.do_solve = P.chain_dags ? 1 : 0;
    sp.chain_blocks = P.chain_blocks ? 1 : 0; sp.n_dags = P.nd;
    sp.dag_done = P.dag_done; sp.sync = x->sync.get<unsigned int>();
    if (x->sync_total > 0x70000000u - (unsigned)P.step_grid) {
      CU(cudaMemsetAsync(sp.sync, 0, sizeof(unsigned int), st));
      x->sync_total = 0;
    }
    sp.sync_target = x->sync_total + (unsigned)P.step_grid;
    sp.n_queries = P.nq;
    sp.in_base = x->dbuf.get(); sp.in_lines = (int64_t)((P.in_bytes + 127) / 128);
    void *args[] = {&sp};
    // step_kernel leaves best_rank / any_in reset for the next launch: no
    // memset, no event between ev[1] and ev[4] (each costs microseconds here)
    cudaError_t le = cudaLaunchCooperativeKernel((const void *)step_kernel, dim3(P.step_grid), dim3(kScanThreads),
                                                 args, P.step_smem, st);
    if (le == cudaSuccess) {
      Launched &L = new_record(P, Path::kFused, P.step_grid);
      L.scan_launches = 1; L.total_launches = 1;
      x->sync_total += (unsigned)P.step_grid;
      P.parity ^= 1;
      if (!P.chain_dags && P.nd) {
        solve_kernel<<<P.nd, kSolveThreads, sizeof(ChainSmem), st>>>(cat->dev, v.in, v.w, v.out, P.task_mv, chain_force_full(), nullptr);
        CU(cudaGetLastError());
        ++L.total_launches;
      }
      CU(cudaEventRecord(x->ev[4], st));
      // one launch: the step is not split into phases (SKYOPT_TRACE has the
      // in-kernel timeline)
      L.scan = L.scan_kernel = {1, 4};
      return 0;
    }
    (void)cudaGetLastError();  // not launched (too large for this device): separate launches below
  }
  Launched &L = new_record(P, Path::kSplit, P.scan2_grid);
  if (P.nq) {
    if (!P.fresh_inputs) {
      CU(cudaMemsetAsync(best_rank, 0xFF, sizeof(uint32_t) * P.nq, st));
      CU(cudaMemsetAsync(any_in, 0, sizeof(uint32_t) * P.nq, st));
    }
    if (P.n_pieces) {
      CU(cudaEventRecord(x->ev[6], st));
      scan2_kernel<<<P.scan2_grid, kScanThreads, P.scan2_smem, st>>>(sa);
      CU(cudaGetLastError());
      CU(cudaEventRecord(x->ev[7], st));
      L.scan_launches = 1; ++L.total_launches;
      L.scan_kernel = {6, 7};
    }
    if (P.finalize) {
      finalize2_kernel<<<(P.nq + 127) / 128, 128, 0, st>>>(cat->dev, cat->fast, P.nq, P.queries,
                                                          best_rank, any_in, P.finals, P.any1);
      CU(cudaGetLastError());
      ++L.total_launches;
    }
  }
  CU(cudaEventRecord(x->ev[2], st));
  L.scan = {1, 2};
  if (!P.solve) return 0;
  if (!P.n_pieces) CU(cudaMemsetAsync(P.err_out, 0, sizeof(int32_t), st));
  if (P.nt) {
    PlaceArgs pa{};
    pa.cat = cat->dev; pa.f = cat->fast; pa.ptasks = P.ptasks; pa.saux = P.saux; pa.best_rank = best_rank;
    pa.any1 = any_in; pa.acc_sets = P.acc_sets; pa.in = v.in; pa.w = v.w;
    pa.task_n = P.task_n; pa.trace = trace; pa.task_mv = nullptr;
    place_kernel<<<P.nt, kScanThreads, sizeof(PlaceSmem), st>>>(pa);
    CU(cudaGetLastError());
    ++L.total_launches;
  }
  CU(cudaEventRecord(x->ev[3], st));
  if (P.nd) {
    solve_kernel<<<P.nd, kSolveThreads, sizeof(ChainSmem), st>>>(cat->dev, v.in, v.w, v.out, P.task_mv, chain_force_full(), nullptr);
    CU(cudaGetLastError());
    ++L.total_launches;
  }
  CU(cudaEventRecord(x->ev[4], st));
  L.expand = {2, 3}; L.solve = {3, 4};
  return 0;
}

// Enqueues the plan's kernels on the context's stream and records in P.ran
// what was launched. Events ev[1..4] bracket the phases.
int enqueue_kernels(SkyoptCatalog *cat, Ctx *x, Plan &P) {
  cudaStream_t st = x->stream;
  if (P.class_tables()) return enqueue_fast(cat, x, P);
  Launched &L = new_record(P, P.path, P.n_blocks);
  CU(cudaEventRecord(x->ev[1], st));
  if (P.nq) {
    CU(cudaMemsetAsync(P.gbest, 0xFF, sizeof(unsigned long long) * P.nsq, st));
    if (P.list_entries) CU(cudaMemsetAsync(P.list_min, 0xFF, sizeof(unsigned long long) * P.list_entries, st));
    if (P.fuzzy_entries) CU(cudaMemsetAsync(P.fuzzy_min, 0xFF, sizeof(unsigned long long) * P.fuzzy_entries, st));
    if (P.n_blocks) {
      ScanArgs sa{};
      sa.cat = cat->dev; sa.squeries = P.squeries; sa.qtests = P.qtests; sa.groups = P.groups;
      sa.n_groups = P.n_groups; sa.partials = P.partials;
      sa.list_min = P.list_min; sa.fuzzy_min = P.fuzzy_min; sa.gbest = P.gbest;
      sa.zero_flag = P.err_out; sa.tile_list = cat->d_tile_list;
      for (int i = 0; i < std::min(P.n_groups, kInlineGroups); ++i) { sa.inline_groups[i] = P.host_groups[i]; sa.inline_block0[i] = P.host_groups[i].block0; }
      sa.n_blocks = P.n_blocks;
      sa.qsplit = 2;
      sa.perm_mul = 1;
      for (uint32_t cand : {7919u, 104729u, 1299709u, 15485863u}) {
        uint64_t x = cand, y = (uint64_t)P.n_blocks;  // gcd
        while (y) { const uint64_t t = x % y; x = y; y = t; }
        if (x == 1) { sa.perm_mul = cand; break; }
      }
      CU(cudaEventRecord(x->ev[6], st));
      if (P.path == Path::kQueue) scan_queue_kernel<<<P.n_blocks, kScanThreads, 0, st>>>(sa);
      else if (P.rpt == 4) scan_kernel<4><<<P.n_blocks, kScanThreads, 0, st>>>(sa);
      else if (P.rpt == 2) scan_kernel<2><<<P.n_blocks, kScanThreads, 0, st>>>(sa);
      else scan_kernel<1><<<P.n_blocks, kScanThreads, 0, st>>>(sa);
      CU(cudaGetLastError());
      CU(cudaEventRecord(x->ev[7], st));
      L.scan_launches = 1; ++L.total_launches;
      L.scan_kernel = {6, 7};
    }
    if (P.finalize) {
      const int fblocks = (P.nq * 32 + 255) / 256;
      finalize_kernel<<<fblocks, 256, 0, st>>>(cat->dev, P.nq, P.partial_base,
                                               P.partial_count, P.partials, P.finals,
                                               P.any1, P.err_out);
      CU(cudaGetLastError());
      ++L.total_launches;
    }
  }
  CU(cudaEventRecord(x->ev[2], st));
  L.scan = {1, 2};
  if (!P.solve) return 0;
  if (!P.n_blocks) CU(cudaMemsetAsync(P.err_out, 0, sizeof(int32_t), st));
  const SolveViews v = solve_views(P);
  if (P.ns) {
    const size_t smem = (size_t)cat->sort_n * 16 + (size_t)cat->max_zones * 8 +
                        (size_t)cat->max_regions * 4;
    expand_kernel<<<P.ns, 128, smem, st>>>(cat->dev, P.slots, P.partial_base,
                                           P.partial_count, P.partials,
                                           P.acc_sets, P.slot_off, cat->sort_n,
                                           cat->max_regions, cat->max_zones, v.ex,
                                           P.err_out);
    CU(cudaGetLastError());
    ++L.total_launches;
  }
  CU(cudaEventRecord(x->ev[3], st));
  if (P.nd) {
    gather_kernel<<<P.nt, kGatherThreads, 0, st>>>(cat->dev, v.in, v.w, P.task_dag, P.task_n, nullptr);
    CU(cudaGetLastError());
    solve_kernel<<<P.nd, kSolveThreads, sizeof(ChainSmem), st>>>(cat->dev, v.in, v.w, v.out, P.task_mv, chain_force_full(), nullptr);
    CU(cudaGetLastError());
    L.total_launches += 2;
  }
  CU(cudaEventRecord(x->ev[4], st));
  L.expand = {2, 3}; L.solve = {3, 4};
  return 0;
}

void fill_scan_results(const SkyoptCatalog *cat, const Plan &P, const Plan &H,
                       SkyoptScanResult *results) {
  (void)cat; (void)P;
  for (int i = 0; i < H.nq; ++i) {
    SkyoptScanResult r{};
    const ScanFinal &f = H.finals[i];
    r.any_stage1 = H.any1[i] ? 1 : 0;
    r.best_row = f.row;
    r.best_inst = f.inst;
    r.best_price = f.row >= 0 ? [&] {
      uint64_t k = f.key;
      uint64_t b = (k & 0x8000000000000000ull) ? (k & 0x7FFFFFFFFFFFFFFFull) : ~k;
      double d; memcpy(&d, &b, 8); return d; }() : NAN;
    results[i] = r;
  }
}

// Host view of the output region, copied back to the start of the pinned buffer.
Plan output_host_view(const Plan &P, char *hbuf) {
  Plan H = P;
  Carver c(hbuf);
  carve_outputs(H, c);
  return H;
}

// One call's round trip on the context's stream: ev[0], the input region to
// the device, the kernels, the output region back, ev[5], and a wait for all
// of it.
int run_plan(SkyoptCatalog *cat, Ctx *x, Plan &P) {
  cudaStream_t st = x->stream;
  CU(cudaEventRecord(x->ev[0], st));
  CU(cudaMemcpyAsync(x->dbuf.get(), x->hbuf.get(), P.in_bytes, cudaMemcpyHostToDevice, st));
  if (int r = enqueue_kernels(cat, x, P)) return r;
  CU(cudaMemcpyAsync(x->hbuf.get(), x->dbuf.get() + P.out_off, P.out_bytes, cudaMemcpyDeviceToHost, st));
  CU(cudaEventRecord(x->ev[5], st));
  CU(cudaStreamSynchronize(st));
  return 0;
}

int copy_solution(SkyoptCatalog *cat, Ctx *x, const Plan &P, const SkyoptProblem *pb,
                  SkyoptSolution *sol) {
  const Plan H = output_host_view(P, x->hbuf.get());
  if (*H.err_out)
    return fail(SKYOPT_ELIMIT, "an instance-type group exceeds the expand capacity (%d rows)", cat->sort_n);
  if (sol->scan) fill_scan_results(cat, P, H, sol->scan);
  if (sol->slot_count && P.ns) memcpy(sol->slot_count, H.slot_count, sizeof(int32_t) * P.ns);
  if (sol->slot_inst && P.ns) memcpy(sol->slot_inst, H.slot_inst, sizeof(int32_t) * P.ns);
  if (sol->chosen && P.nt) memcpy(sol->chosen, H.chosen, sizeof(SkyoptCandidate) * P.nt);
  if (sol->chosen_index && P.nt) memcpy(sol->chosen_index, H.chosen_index, sizeof(int32_t) * P.nt);
  if (sol->task_n_candidates && P.nt) memcpy(sol->task_n_candidates, H.task_n, sizeof(int32_t) * P.nt);
  if (sol->dag && P.nd) memcpy(sol->dag, H.dagres, sizeof(SkyoptDagResult) * P.nd);
  // Tasks of a failed DAG carry no plan.
  if (sol->chosen_index) {
    for (int d = 0; d < P.nd; ++d)
      if (H.dagres[d].status != 0)
        for (int t = pb->dags[d].task_begin; t < pb->dags[d].task_end; ++t) {
          sol->chosen_index[t] = -1;
          if (sol->chosen) { sol->chosen[t] = SkyoptCandidate{}; sol->chosen[t].slot = -1; sol->chosen[t].inst_id = -1; }
        }
  }
  if (sol->cand_cap > 0 && sol->candidates && sol->task_cand_offset) {
    std::vector<int64_t> off(P.nt + 1, 0);
    for (int t = 0; t < P.nt; ++t) off[t + 1] = off[t] + H.task_n[t];
    if (off[P.nt] > sol->cand_cap)
      return fail(SKYOPT_ELIMIT, "candidate table needs %lld entries, capacity %lld",
                  (long long)off[P.nt], (long long)sol->cand_cap);
    memcpy(sol->task_cand_offset, off.data(), sizeof(int64_t) * (P.nt + 1));
    if (off[P.nt] > 0) {
      int64_t *d_off; SkyoptCandidate *d_tab;
      if (int rc = carve_in(x->scratch, x->stream, [&](Carver &c) {
            d_off = c.take<int64_t>(P.nt + 1);
            d_tab = c.take<SkyoptCandidate>(off[P.nt]);
          }))
        return rc;
      CU(cudaMemcpyAsync(d_off, off.data(), sizeof(int64_t) * (P.nt + 1), cudaMemcpyHostToDevice, x->stream));
      const SolveViews v = solve_views(P);
      table_kernel<<<P.nt, 128, 0, x->stream>>>(v.in, v.w, P.task_n, P.nt, d_off, d_tab);
      CU(cudaGetLastError());
      CU(cudaMemcpyAsync(sol->candidates, d_tab, sizeof(SkyoptCandidate) * off[P.nt],
                         cudaMemcpyDeviceToHost, x->stream));
      CU(cudaStreamSynchronize(x->stream));
    }
  }
  return 0;
}

// The time between the events of `s`, if it names any.
int elapsed(Ctx *x, Launched::Span s, float *ms) {
  if (s.begin != s.end) CU(cudaEventElapsedTime(ms, x->ev[s.begin], x->ev[s.end]));
  return 0;
}

// SkyoptStats of a call: the record of what it launched, its phase times and
// its total from ev[0] to ev[5].
int fill_stats(Ctx *x, const Launched &L, SkyoptStats *stats) {
  if (!stats) return 0;
  memset(stats, 0, sizeof(*stats));
  int r;
  if ((r = elapsed(x, L.scan, &stats->scan_ms)) || (r = elapsed(x, L.expand, &stats->expand_ms)) ||
      (r = elapsed(x, L.solve, &stats->solve_ms)) || (r = elapsed(x, L.scan_kernel, &stats->scan_kernel_ms)) ||
      (r = elapsed(x, {0, 5}, &stats->total_ms)))
    return r;
  stats->scan_launches = L.scan_launches;
  stats->total_launches = L.total_launches;
  stats->scan_rows = L.scan_rows;
  stats->scan_passes_rows = L.pass_rows;
  stats->scan_blocks = L.scan_blocks;
  stats->scan_form = (int32_t)L.form;
  stats->reserved_ = (int32_t)std::min<int64_t>(L.layout_rows, 0x7FFFFFFF);
  return 0;
}

// Plan, run and read back one optimisation (skyopt_optimize,
// skyopt_session_open). `P` stays valid after the call.
int optimize_once(SkyoptCatalog *cat, Ctx *x, const SkyoptProblem *pb, const int32_t *rr,
                  int nrr, SkyoptSolution *sol, SkyoptStats *stats, Plan &P) {
  int r = build_plan(cat, pb, x, true, sol->scan != nullptr, P, rr, nrr);
  if (r) return r;
  if ((r = run_plan(cat, x, P))) return r;
  if ((r = copy_solution(cat, x, P, pb, sol))) return r;
  return fill_stats(x, P.ran, stats);
}

// skyopt_solve_tables' device arrays and their sizes.
struct TablePlan {
  int64_t total;  // candidates
  int nt, np, ntar, nd, nc;
  double *values, *tariffs, *dp;
  int32_t *clouds, *parents, *task_n, *back, *chosen_index;
  int64_t *task_off;
  SkyoptTask *tasks;
  SkyoptDag *dags;
  SkyoptDagResult *results;
  TaskMin *task_mv;
};

void carve_tables(TablePlan &T, Carver &c) {
  T.values = c.take<double>(T.total);
  T.clouds = c.take<int32_t>(T.total);
  T.task_off = c.take<int64_t>(T.nt + 1);
  T.tasks = c.take<SkyoptTask>(T.nt);
  T.parents = c.take<int32_t>(T.np);
  T.tariffs = c.take<double>(T.ntar);
  T.dags = c.take<SkyoptDag>(T.nd);
  T.task_n = c.take<int32_t>(T.nt);
  T.dp = c.take<double>(T.total);
  T.back = c.take<int32_t>(T.total);
  T.chosen_index = c.take<int32_t>(T.nt);
  T.results = c.take<SkyoptDagResult>(T.nd);
  T.task_mv = c.take<TaskMin>((size_t)T.nt * T.nc);
}

}  // namespace

extern "C" {

static_assert(sizeof(SkyoptStats) == 56 && offsetof(SkyoptStats, scan_form) == 48, "SkyoptStats ABI");
int skyopt_abi_version(void) { return SKYOPT_ABI_VERSION; }
int skyopt_dag_kinds(void) { return SKYOPT_DAG_SAME_INFRA; }

uint64_t skyopt_price_key(double price) {
  uint64_t b; memcpy(&b, &price, 8);
  return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
}
const char *skyopt_last_error(void) { return g_error.c_str(); }

int skyopt_device_count(int *count) {
  if (!count) return fail(SKYOPT_EINVAL, "count is NULL");
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess) { *count = 0; return fail(SKYOPT_ENODEV, "cudaGetDeviceCount: %s", cudaGetErrorString(e)); }
  *count = n;
  return 0;
}

int skyopt_catalog_create(const SkyoptCatalogDesc *d, int device, SkyoptCatalog **out) {
  NvtxRange nvtx_("skyopt_catalog_create");
  if (!d || !out) return fail(SKYOPT_EINVAL, "NULL argument");
  *out = nullptr;
  if (d->n_rows <= 0 || d->n_rows % kZoneRows != 0) return fail(SKYOPT_EINVAL, "n_rows must be a positive multiple of 128");
  if (d->n_rows > 0x7FFFFFF0ll) return fail(SKYOPT_ELIMIT, "catalog exceeds 2^31 rows");
  if (d->n_clouds <= 0 || d->n_clouds > SKYOPT_MAX_CLOUDS) return fail(SKYOPT_ELIMIT, "1..%d clouds supported", SKYOPT_MAX_CLOUDS);
  if (d->n_acc_keys < 0 || d->n_acc_keys > 32 * SKYOPT_ACC_SET_WORDS)
    return fail(SKYOPT_ELIMIT, "at most %d distinct (accelerator, count) pairs", 32 * SKYOPT_ACC_SET_WORDS);
  if (!d->price || !d->spot_price || !d->vcpus || !d->mem || !d->acc_key || !d->region_id ||
      !d->zone_id || !d->flags || !d->inst_id || !d->cloud_row_offsets || !d->cloud_inst_offsets ||
      !d->cloud_region_offsets || !d->cloud_n_zones || !d->region_is_us || !d->inst_row_offsets ||
      !d->inst_rows || !d->acc_row_offsets || !d->acc_rows || !d->inst_acc_key || !d->zone_map)
    return fail(SKYOPT_EINVAL, "a required column pointer is NULL");
  if (d->cloud_row_offsets[0] != 0 || d->cloud_row_offsets[d->n_clouds] != d->n_rows)
    return fail(SKYOPT_EINVAL, "cloud_row_offsets must span [0, n_rows]");
  for (int c = 0; c < d->n_clouds; ++c)
    if (d->cloud_row_offsets[c] % kZoneRows != 0 || d->cloud_row_offsets[c + 1] < d->cloud_row_offsets[c])
      return fail(SKYOPT_EINVAL, "cloud %d row range must be 128-row aligned", c);
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0)
    return fail(SKYOPT_ENODEV, "no CUDA device available; libskyopt has no CPU fallback");
  if (device < 0 || device >= ndev) return fail(SKYOPT_EINVAL, "device %d out of range (%d devices)", device, ndev);
  CU(cudaSetDevice(device));
  // destroyed on every return until it is handed out
  std::unique_ptr<SkyoptCatalog, int (*)(SkyoptCatalog *)> owner(new (std::nothrow) SkyoptCatalog(),
                                                                  skyopt_catalog_destroy);
  if (!owner) return fail(SKYOPT_ENOMEM, "out of host memory");
  SkyoptCatalog *c = owner.get();
  c->device = device;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) {
    c->sm_count = prop.multiProcessorCount;
    c->l2_bytes = prop.l2CacheSize;
  }

  const size_t n = (size_t)d->n_rows;
  const size_t slack = kOverReadRows;
  int rc = 0;
  CatDev &v = c->dev;
  v.n_rows = d->n_rows;
  v.n_clouds = d->n_clouds; v.n_inst = d->n_inst; v.n_acc_keys = d->n_acc_keys; v.n_regions = d->n_regions;
  const size_t n_inst_rows = (size_t)d->inst_row_offsets[d->n_inst];
  const size_t n_acc_rows = (size_t)d->acc_row_offsets[d->n_acc_keys];
  rc = rc ? rc : upload(c, d->price, n, slack, &v.price);
  rc = rc ? rc : upload(c, d->spot_price, n, slack, &v.spot);
  rc = rc ? rc : upload(c, d->vcpus, n, slack, &v.vcpus);
  rc = rc ? rc : upload(c, d->mem, n, slack, &v.mem);
  if (d->disk_total) rc = rc ? rc : upload(c, d->disk_total, n, slack, &v.disk_total);
  rc = rc ? rc : upload(c, d->acc_key, n, slack, &v.acc_key, 0xFF);
  rc = rc ? rc : upload(c, d->region_id, n, slack, &v.region_id);
  rc = rc ? rc : upload(c, d->zone_id, n, slack, &v.zone_id, 0xFF);
  rc = rc ? rc : upload(c, d->flags, n, slack, &v.flags);
  rc = rc ? rc : upload(c, d->inst_id, n, slack, &v.inst_id, 0xFF);
  rc = rc ? rc : upload(c, d->cloud_row_offsets, (size_t)d->n_clouds + 1, 0, &v.cloud_row_offsets);
  rc = rc ? rc : upload(c, d->cloud_inst_offsets, (size_t)d->n_clouds + 1, 0, &v.cloud_inst_offsets);
  rc = rc ? rc : upload(c, d->cloud_region_offsets, (size_t)d->n_clouds + 1, 0, &v.cloud_region_offsets);
  rc = rc ? rc : upload(c, d->cloud_n_zones, (size_t)d->n_clouds, 0, &v.cloud_n_zones);
  rc = rc ? rc : upload(c, d->region_is_us, (size_t)std::max(d->n_regions, 1), 0, &v.region_is_us);
  rc = rc ? rc : upload(c, d->inst_row_offsets, (size_t)d->n_inst + 1, 0, &v.inst_row_offsets);
  rc = rc ? rc : upload(c, d->inst_rows, n_inst_rows, 1, &v.inst_rows);
  rc = rc ? rc : upload(c, d->acc_row_offsets, (size_t)d->n_acc_keys + 1, 0, &v.acc_row_offsets);
  rc = rc ? rc : upload(c, d->acc_rows, n_acc_rows, 1, &v.acc_rows);
  rc = rc ? rc : upload(c, d->inst_acc_key, (size_t)std::max(d->n_inst, 1), 0, &v.inst_acc_key, 0xFF);
  static_assert(sizeof(SkyoptZone) == sizeof(RowSummary), "zone map ABI");
  rc = rc ? rc : upload(c, reinterpret_cast<const RowSummary *>(d->zone_map), n / kZoneRows,
                        kOverReadRows / kZoneRows + 1, &v.zone_map);
  if (rc) return rc;
  for (int64_t z = 0; z < n / kZoneRows; ++z) {
    const RowSummary &r = reinterpret_cast<const RowSummary *>(d->zone_map)[z];
    c->zm_flags.push_back(r.fl_or); c->zm_grp.push_back(r.grp);
    c->zm_sig_lo.push_back(r.sg_lo); c->zm_sig_hi.push_back(r.sg_hi);
  }

  {
    std::vector<int32_t> tile_list;
    for (int r = 0; r < 3; ++r) {
      const int cpt = 2 << r;  // 128-row chunks per tile
      c->tile_class[r].assign(d->n_clouds, {});
      for (int cl = 0; cl < d->n_clouds; ++cl) {
        const int64_t z0 = d->cloud_row_offsets[cl] / kZoneRows, z1 = d->cloud_row_offsets[cl + 1] / kZoneRows;
        const int n_tiles = (int)((z1 - z0 + cpt - 1) / cpt);
        std::vector<int32_t> members[2];
        std::array<int64_t, 256> exact[2] = {};
        int64_t chunks[2] = {0, 0};
        for (int t = 0; t < n_tiles; ++t) {
          int with_default = 0, n = 0;
          for (int64_t z = z0 + (int64_t)t * cpt; z < std::min<int64_t>(z1, z0 + (int64_t)(t + 1) * cpt); ++z, ++n)
            with_default += (d->zone_map[z].flags_or & SKYOPT_F_DEFAULT_FAMILY) ? 1 : 0;
          const int k = (with_default * 4 >= n) ? 1 : 0;
          members[k].push_back(t);
          for (int64_t z = z0 + (int64_t)t * cpt; z < std::min<int64_t>(z1, z0 + (int64_t)(t + 1) * cpt); ++z)
            exact[k][d->zone_map[z].flags_or & 0xFFu]++;
          chunks[k] += n;
        }
        for (int k = 0; k < 2; ++k) {
          SkyoptCatalog::TileClass &tc = c->tile_class[r][cl][k];
          tc.n_tiles = (int)members[k].size();
          if (tc.n_tiles > 0) {
            tc.tile0 = members[k].front();
            if (members[k].back() - members[k].front() + 1 != tc.n_tiles) {
              tc.list0 = (int)tile_list.size();
              tile_list.insert(tile_list.end(), members[k].begin(), members[k].end());
            }
          }
          for (int m = 0; m < 256; ++m) {
            int64_t n = 0;
            for (int f = 0; f < 256; ++f) if ((f & m) == m) n += exact[k][f];
            tc.density[m] = chunks[k] ? (float)((double)n / (double)chunks[k]) : 0.f;
          }
        }
      }
    }
    if (tile_list.empty()) tile_list.push_back(0);
    rc = upload(c, tile_list.data(), tile_list.size(), 0, &c->d_tile_list);
    if (rc) return rc;
  }
  c->cloud_row_offsets.assign(d->cloud_row_offsets, d->cloud_row_offsets + d->n_clouds + 1);
  c->cloud_inst_offsets.assign(d->cloud_inst_offsets, d->cloud_inst_offsets + d->n_clouds + 1);
  c->cloud_region_offsets.assign(d->cloud_region_offsets, d->cloud_region_offsets + d->n_clouds + 1);
  c->cloud_n_zones.assign(d->cloud_n_zones, d->cloud_n_zones + d->n_clouds);
  // Expand capacity per cloud: largest instance-type group, or all
  // accelerator-only rows of one key.
  c->cloud_group_cap.assign(d->n_clouds, 1);
  int max_group = 1;
  for (int cl = 0; cl < d->n_clouds; ++cl) {
    int cap = 1;
    for (int i = d->cloud_inst_offsets[cl]; i < d->cloud_inst_offsets[cl + 1]; ++i)
      cap = std::max(cap, d->inst_row_offsets[i + 1] - d->inst_row_offsets[i]);
    c->cloud_group_cap[cl] = cap;
    c->max_regions = std::max(c->max_regions, d->cloud_region_offsets[cl + 1] - d->cloud_region_offsets[cl]);
    c->max_zones = std::max(c->max_zones, d->cloud_n_zones[cl]);
  }
  // accelerator groups may span clouds in the CSR; bound them by the group
  for (int k = 0; k < d->n_acc_keys; ++k) {
    const int rows = d->acc_row_offsets[k + 1] - d->acc_row_offsets[k];
    if (!rows) continue;
    // an exact accelerator set may union a few keys (case variants): x4 slack
    for (int cl = 0; cl < d->n_clouds; ++cl) {
      bool in_cloud = false;
      for (int i = d->acc_row_offsets[k]; i < d->acc_row_offsets[k + 1] && !in_cloud; ++i)
        in_cloud = d->acc_rows[i] >= d->cloud_row_offsets[cl] && d->acc_rows[i] < d->cloud_row_offsets[cl + 1];
      if (in_cloud) c->cloud_group_cap[cl] = std::max(c->cloud_group_cap[cl], rows);
    }
  }
  for (int cl = 0; cl < d->n_clouds; ++cl) max_group = std::max(max_group, c->cloud_group_cap[cl]);
  if (max_group > SKYOPT_MAX_GROUP_ROWS)
    return fail(SKYOPT_ELIMIT, "an instance type has %d rows; the limit is %d", max_group, SKYOPT_MAX_GROUP_ROWS);
  c->sort_n = std::max(2, next_pow2(max_group));
  for (int cl = 0; cl < d->n_clouds; ++cl) c->cloud_group_cap[cl] = c->sort_n;  // sorted output is written sparsely
  const size_t smem = (size_t)c->sort_n * 16 + (size_t)c->max_zones * 8 + (size_t)c->max_regions * 4;
  if (smem > 200 * 1024) return fail(SKYOPT_ELIMIT, "expand needs %zu B of shared memory", smem);
  // The attribute is per function, not per catalog: only ever raise it.
  static std::mutex attr_mu;
  static size_t attr_expand = 48 * 1024;
  cudaError_t e = cudaSuccess;
  {
    std::lock_guard<std::mutex> g(attr_mu);
    if (smem > attr_expand) {
      e = cudaFuncSetAttribute(expand_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (e == cudaSuccess) attr_expand = smem;
    }
  }
  if (e != cudaSuccess) return fail(SKYOPT_ECUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
  e = cudaFuncSetAttribute(solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ChainSmem));
  if (e != cudaSuccess) return fail(SKYOPT_ECUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
  rc = build_fast(c, d);
  if (rc) return rc;
  if (c->fast_ok) {
    int coop = 0;
    if (cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, device) == cudaSuccess) c->coop = coop != 0;
    e = cudaFuncSetAttribute(step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(place_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(PlaceSmem));
    if (e == cudaSuccess)
    e = cudaFuncSetAttribute(scan2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
    if (e != cudaSuccess) return fail(SKYOPT_ECUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
  }
  CU(cudaDeviceSynchronize());
  *out = owner.release();
  return 0;
}

int skyopt_catalog_destroy(SkyoptCatalog *c) {
  if (!c) return 0;
  cudaSetDevice(c->device);
  for (Ctx *x : c->free_ctx) delete x;
  for (void *p : c->allocs) cudaFree(p);
  delete c;
  return 0;
}

int skyopt_catalog_set_scan_mode(SkyoptCatalog *c, int mode) {
  if (!c || mode < 0 || mode > 9)
    return fail(SKYOPT_EINVAL, "scan mode must be 0 (auto), 1 (tile), "
                               "4 (queue), 5 (queue, 32 tiles per block), 7 (class-table scan, one fused launch, "
                               "without pruning), 8 (class-table scan as separate launches) or 9 (8 without pruning)");
  if (mode == 2 || mode == 3)
    return fail(SKYOPT_EINVAL, "scan modes 2 and 3 (the TMA streaming scan) were removed");
  if (mode == 6)
    return fail(SKYOPT_EINVAL, "scan mode 6 was removed: mode 0 (auto) runs the same kernels");
  if (mode >= 7 && !c->fast_ok) return fail(SKYOPT_ELIMIT, "the class-table scan is not available for this catalog");
  c->scan_mode = mode;
  return 0;
}

int skyopt_set_chain_paths(int flags) {
  if (flags & ~(SKYOPT_CHAIN_FULL | SKYOPT_CHAIN_GENERAL | SKYOPT_CHAIN_LAST_TASK_BLOCK))
    return fail(SKYOPT_EINVAL, "unknown chain path flags 0x%x", flags);
  g_chain_paths.store(flags, std::memory_order_relaxed);
  return 0;
}

int skyopt_set_scan_pieces(int flags) {
  if (flags & ~SKYOPT_SCAN_PIECES_EQUAL) return fail(SKYOPT_EINVAL, "unknown scan piece flags 0x%x", flags);
  g_scan_pieces.store(flags, std::memory_order_relaxed);
  return 0;
}

int skyopt_scan_pieces(SkyoptCatalog *cat, const SkyoptProblem *pb, int fused, SkyoptScanPiece *out, int cap,
                       int *n_pieces, int *n_groups, int *grid, int32_t *q_begin, int32_t *q_count,
                       int32_t *order_out) {
  if (!cat || !pb || !out || cap < 0 || !n_pieces || !n_groups || !grid) return fail(SKYOPT_EINVAL, "bad arguments");
  int rc = validate_problem(cat, pb);
  if (rc) return rc;
  if (!takes_class_tables(cat, pb)) return fail(SKYOPT_ELIMIT, "the class-table scan does not take this problem");
  CU(cudaSetDevice(cat->device));  // group_class_tables asks the device for occupancy
  Plan P;
  P.nq = pb->n_queries; P.ns = pb->n_slots; P.nt = pb->n_tasks; P.nd = pb->n_dags;
  P.noprune = cat->scan_mode == 7 || cat->scan_mode == 9;
  P.path = fused ? Path::kFused : Path::kSplit;
  std::vector<std::vector<int>> by_cloud(cat->dev.n_clouds);
  for (int i = 0; i < P.nq; ++i) by_cloud[pb->queries[i].cloud].push_back(i);
  std::vector<Scan2Group> groups2;
  std::vector<int> order2;
  group_class_tables(cat, pb, by_cloud, P, groups2, order2);
  if (P.n_pieces > cap || P.n_groups2 > cap) return fail(SKYOPT_ELIMIT, "%d pieces, %d groups: more than %d", P.n_pieces, P.n_groups2, cap);
  const int launch_grid = fused ? P.step_grid : P.scan2_grid;
  for (const Scan2Group &G : groups2) {
    // the kernel's slice rule: shared tables only in the cooperative launch
    const bool shared = fused && G.n_pieces > 1 && P.n_pieces <= launch_grid;
    const int n_all = G.n_fa + G.n_cm + G.n_rz;
    for (int pi = 0; pi < G.n_pieces; ++pi) {
      SkyoptScanPiece &o = out[G.piece0 + pi];
      o.group = G.index; o.cloud = G.cloud; o.col = G.col;
      o.chunk_begin = P.piece_chunk0[G.piece0 + pi];
      o.chunk_end = pi + 1 < G.n_pieces ? P.piece_chunk0[G.piece0 + pi + 1] : G.chunk0 + G.n_chunks;
      o.slice_entries = shared ? (int)((int64_t)n_all * (pi + 1) / G.n_pieces) - (int)((int64_t)n_all * pi / G.n_pieces)
                               : n_all;
    }
    if (q_begin) q_begin[G.index] = G.q_begin;
    if (q_count) q_count[G.index] = G.q_count;
  }
  if (order_out) std::copy(order2.begin(), order2.end(), order_out);
  *n_pieces = P.n_pieces; *n_groups = P.n_groups2; *grid = launch_grid;
  return 0;
}

int skyopt_catalog_bytes(const SkyoptCatalog *c, int64_t *device_bytes, int64_t *row_bytes) {
  if (!c) return fail(SKYOPT_EINVAL, "NULL catalog");
  if (device_bytes) *device_bytes = c->device_bytes;
  // bytes the scan streams per row and pass: one price column, vCPUs,
  // MemoryGiB (f64) + acc_key, region, zone, flags (u16)
  if (row_bytes) *row_bytes = 3 * 8 + 4 * 2;
  return 0;
}

int skyopt_list_offerings(SkyoptCatalog *cat, int cloud, int by_acc_key,
                          const int32_t *group_ids, int n_groups,
                          const uint32_t *region_mask, int per_region,
                          int32_t *out_rows) {
  NvtxRange nvtx_("skyopt_list_offerings");
  if (!cat || !group_ids || !out_rows || n_groups <= 0) return fail(SKYOPT_EINVAL, "bad arguments");
  if (cloud < 0 || cloud >= cat->dev.n_clouds) return fail(SKYOPT_EINVAL, "cloud %d out of range", cloud);
  const int n_max = by_acc_key ? cat->dev.n_acc_keys : cat->dev.n_inst;
  for (int i = 0; i < n_groups; ++i)
    if (group_ids[i] < 0 || group_ids[i] >= n_max) return fail(SKYOPT_EINVAL, "group %d: id %d out of range", i, group_ids[i]);
  const int n_regions = cat->cloud_region_offsets[cloud + 1] - cat->cloud_region_offsets[cloud];
  const int slots = per_region ? std::max(n_regions, 1) : 1;
  const size_t smem = (size_t)slots * 20 + 8;
  if (smem > 48 * 1024) return fail(SKYOPT_ELIMIT, "cloud has too many regions (%d)", n_regions);
  Lease x;
  if (int rc = x.open(cat)) return rc;
  cudaStream_t st = x->stream;
  int32_t *d_ids, *d_out; uint32_t *d_mask;
  const int mask_words = (std::max(n_regions, 1) + 31) / 32;
  if (int rc = carve_in(x->scratch, st, [&](Carver &c) {
        d_ids = c.take<int32_t>(n_groups);
        d_out = c.take<int32_t>((size_t)n_groups * slots);
        d_mask = region_mask ? c.take<uint32_t>(mask_words) : nullptr;
      }))
    return rc;
  CU(cudaMemcpyAsync(d_ids, group_ids, sizeof(int32_t) * (size_t)n_groups, cudaMemcpyHostToDevice, st));
  if (region_mask)
    CU(cudaMemcpyAsync(d_mask, region_mask, sizeof(uint32_t) * (size_t)mask_words, cudaMemcpyHostToDevice, st));
  offer_kernel<<<n_groups, 128, smem, st>>>(cat->dev, cloud, by_acc_key ? 1 : 0, d_ids, d_mask,
                                            per_region ? 1 : 0, std::max(n_regions, 1), d_out);
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(out_rows, d_out, sizeof(int32_t) * (size_t)n_groups * slots, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return x.finish(0);
}

static_assert(sizeof(SkyoptPriceQuery) == 24, "SkyoptPriceQuery ABI");

int skyopt_price(SkyoptCatalog *cat, const SkyoptPriceQuery *q, int n, double *hourly, int32_t *status) {
  NvtxRange nvtx_("skyopt_price");
  if (!cat || n < 0 || (n > 0 && (!q || !hourly || !status))) return fail(SKYOPT_EINVAL, "bad arguments");
  for (int i = 0; i < n; ++i) {
    const SkyoptPriceQuery &r = q[i];
    if (r.kind != SKYOPT_PRICE_INSTANCE && r.kind != SKYOPT_PRICE_ACCELERATOR)
      return fail(SKYOPT_EINVAL, "request %d: kind %d", i, r.kind);
    if (r.cloud < 0 || r.cloud >= cat->dev.n_clouds) return fail(SKYOPT_EINVAL, "request %d: cloud %d out of range", i, r.cloud);
    const int c = r.cloud;
    const bool id_ok = r.kind == SKYOPT_PRICE_INSTANCE
                           ? r.id >= cat->cloud_inst_offsets[c] && r.id < cat->cloud_inst_offsets[c + 1]
                           : r.id >= 0 && r.id < cat->dev.n_acc_keys;
    if (!id_ok) return fail(SKYOPT_EINVAL, "request %d: id %d out of range", i, r.id);
    if (r.price_col != 0 && r.price_col != 1) return fail(SKYOPT_EINVAL, "request %d: price column %d", i, r.price_col);
    const int n_regions = cat->cloud_region_offsets[c + 1] - cat->cloud_region_offsets[c];
    if (r.region_id < -1 || r.region_id >= n_regions)
      return fail(SKYOPT_EINVAL, "request %d: region %d out of range", i, r.region_id);
    if (r.zone_id < -1 || r.zone_id >= cat->cloud_n_zones[c])
      return fail(SKYOPT_EINVAL, "request %d: zone %d out of range", i, r.zone_id);
  }
  if (n == 0) return 0;
  Lease x;
  if (int rc = x.open(cat)) return rc;
  cudaStream_t st = x->stream;
  SkyoptPriceQuery *d_q; double *d_hourly; int32_t *d_status;
  if (int rc = carve_in(x->scratch, st, [&](Carver &c) {
        d_q = c.take<SkyoptPriceQuery>(n);
        d_hourly = c.take<double>(n);  // the two outputs: one D2H copy
        d_status = c.take<int32_t>(n);
      }))
    return rc;
  const size_t status_off = (size_t)((char *)d_status - (char *)d_hourly);
  const size_t out_bytes = status_off + sizeof(int32_t) * (size_t)n;
  if (int rc = x->hbuf.reserve(out_bytes, st)) return rc;
  CU(cudaMemcpyAsync(d_q, q, sizeof(SkyoptPriceQuery) * (size_t)n, cudaMemcpyHostToDevice, st));
  const int warps_per_block = kPriceThreads / 32;
  price_kernel<<<(unsigned)((n + warps_per_block - 1) / warps_per_block), kPriceThreads, 0, st>>>(
      cat->dev, d_q, n, d_hourly, d_status);
  CU(cudaGetLastError());
  char *h = x->hbuf.get();
  CU(cudaMemcpyAsync(h, d_hourly, out_bytes, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  memcpy(hourly, h, sizeof(double) * (size_t)n);
  memcpy(status, h + status_off, sizeof(int32_t) * (size_t)n);
  return x.finish(0);
}

int skyopt_scan(SkyoptCatalog *cat, const SkyoptQuery *queries, int n_queries,
                const uint32_t *acc_sets, int n_acc_sets, SkyoptScanResult *results,
                int32_t *list_ids, double *list_prices, int list_cap,
                int32_t *fuzzy_keys, double *fuzzy_prices, int fuzzy_cap,
                SkyoptStats *stats) {
  NvtxRange nvtx_("skyopt_scan");
  if (!cat || !queries || !results || n_queries <= 0) return fail(SKYOPT_EINVAL, "bad arguments");
  if (list_cap > 2048 || fuzzy_cap > 2048) return fail(SKYOPT_ELIMIT, "list capacity is limited to 2048 entries");
  SkyoptProblem pb{};
  pb.queries = queries; pb.n_queries = n_queries; pb.acc_sets = acc_sets; pb.n_acc_sets = n_acc_sets;
  int rc = validate_problem(cat, &pb);
  if (rc) return rc;
  Lease x;
  if ((rc = x.open(cat))) return rc;
  Plan P;
  const bool want_list = list_ids && list_prices && list_cap > 0;
  const bool want_fuzzy = fuzzy_keys && fuzzy_prices && fuzzy_cap > 0;
  if ((rc = build_plan(cat, &pb, x.ctx(), false, true, P))) return rc;
  if ((rc = run_plan(cat, x.ctx(), P))) return rc;
  cudaStream_t st = x->stream;
  fill_scan_results(cat, P, output_host_view(P, x->hbuf.get()), results);
  for (int kind = 0; kind < 2; ++kind) {
    const bool want = kind == 0 ? want_list : want_fuzzy;
    if (!want) continue;
    const int cap = kind == 0 ? list_cap : fuzzy_cap;
    const int n_entries_max = kind == 0 ? cat->dev.n_inst : cat->dev.n_acc_keys;
    const int sort_n = std::min(2048, std::max(2, next_pow2(std::max(n_entries_max, cap))));
    int32_t *d_ids, *d_cnt; double *d_pr;
    if ((rc = carve_in(x->scratch, st, [&](Carver &c) {
           d_ids = c.take<int32_t>((size_t)n_queries * cap);
           d_pr = c.take<double>((size_t)n_queries * cap);
           d_cnt = c.take<int32_t>(n_queries);
         })))
      return rc;
    list_kernel<<<n_queries, 256, (size_t)sort_n * 16, st>>>(
        cat->dev, P.queries, kind, kind == 0 ? P.list_base : P.fuzzy_base,
        kind == 0 ? P.list_min : P.fuzzy_min, cap, sort_n, d_ids, d_pr, d_cnt);
    CU(cudaGetLastError());
    std::vector<int32_t> cnt(n_queries);
    CU(cudaMemcpyAsync(kind == 0 ? list_ids : fuzzy_keys, d_ids, sizeof(int32_t) * (size_t)n_queries * cap, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(kind == 0 ? list_prices : fuzzy_prices, d_pr, sizeof(double) * (size_t)n_queries * cap, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(cnt.data(), d_cnt, sizeof(int32_t) * (size_t)n_queries, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    for (int i = 0; i < n_queries; ++i) (kind == 0 ? results[i].n_list : results[i].n_fuzzy) = cnt[i];
  }
  return x.finish(fill_stats(x.ctx(), P.ran, stats));
}

int skyopt_optimize(SkyoptCatalog *cat, const SkyoptProblem *pb, SkyoptSolution *sol,
                    SkyoptStats *stats) {
  return skyopt_optimize_blocks(cat, pb, nullptr, 0, sol, stats);
}

int skyopt_optimize_blocks(SkyoptCatalog *cat, const SkyoptProblem *pb, const int32_t *rr, int nrr,
                           SkyoptSolution *sol, SkyoptStats *stats) {
  NvtxRange nvtx_("skyopt_optimize");
  if (!cat || !pb || !sol) return fail(SKYOPT_EINVAL, "NULL argument");
  if (pb->n_dags <= 0 || pb->n_tasks <= 0 || pb->n_slots <= 0)
    return fail(SKYOPT_EINVAL, "empty problem");
  int rc = validate_problem(cat, pb, rr, nrr);
  if (rc) return rc;
  Lease x;
  if ((rc = x.open(cat))) return rc;
  Plan P;
  return x.finish(optimize_once(cat, x.ctx(), pb, rr, nrr, sol, stats, P));
}

struct SkyoptSession {
  Lease lease;                       // the session's context, from open to close
  Plan P;
  std::vector<SkyoptDag> dags;       // host copy: task ranges, flags, blocked ranges
  DeviceBuffer d_blocked, d_dags;
  std::vector<int32_t> ids;          // a re-solve's tasks, then its DAGs
  DeviceBuffer d_ids;
  // skyopt_session_update_dags: every slot's reservation flag and task's
  // slot range (host copies), the reservation tables (the current one and
  // the incoming one; P.resv / P.resv_off point at the current one once an
  // update ran, before that at the problem's input region), the incoming
  // flags, the re-priced tasks and the per-DAG marks
  std::vector<int32_t> pad, task_slots, marks;
  DeviceBuffer d_resv[2], d_resv_off[2];
  int cur = -1;
  DeviceBuffer d_pad, d_marks, d_tasks;
};

int skyopt_session_open(SkyoptCatalog *cat, const SkyoptProblem *pb, SkyoptSolution *sol,
                        SkyoptStats *stats, SkyoptSession **out) {
  return skyopt_session_open_blocks(cat, pb, nullptr, 0, sol, stats, out);
}

int skyopt_session_open_blocks(SkyoptCatalog *cat, const SkyoptProblem *pb, const int32_t *rr,
                               int nrr, SkyoptSolution *sol, SkyoptStats *stats,
                               SkyoptSession **out) {
  NvtxRange nvtx_("skyopt_session_open");
  if (!cat || !pb || !sol || !out) return fail(SKYOPT_EINVAL, "NULL argument");
  *out = nullptr;
  if (pb->n_dags <= 0 || pb->n_tasks <= 0 || pb->n_slots <= 0)
    return fail(SKYOPT_EINVAL, "empty problem");
  int rc = validate_problem(cat, pb, rr, nrr);
  if (rc) return rc;
  std::unique_ptr<SkyoptSession> s(new (std::nothrow) SkyoptSession());
  if (!s) return fail(SKYOPT_ENOMEM, "out of host memory");
  if ((rc = s->lease.open(cat))) return rc;
  if ((rc = s->lease.finish(optimize_once(cat, s->lease.ctx(), pb, rr, nrr, sol, stats, s->P)))) return rc;
  s->dags.assign(pb->dags, pb->dags + pb->n_dags);
  s->pad.resize(pb->n_slots);
  for (int i = 0; i < pb->n_slots; ++i) s->pad[i] = pb->slots[i].pad_;
  s->task_slots.resize(2 * (size_t)pb->n_tasks);
  for (int t = 0; t < pb->n_tasks; ++t) {
    s->task_slots[2 * t] = pb->tasks[t].slot_begin;
    s->task_slots[2 * t + 1] = pb->tasks[t].slot_end;
  }
  *out = s.release();
  return 0;
}

// A session call's list of DAGs: `ids[k]` names a DAG of the session, none
// twice (`listed` returns which are listed), and each DAG's blocked range
// lies inside [0, n_blocked]. The ranges are `ranges[2k], ranges[2k + 1]`
// of DAG ids[k], or with `every_dag` those of DAG k for every DAG.
// `name` / `verb`: the list's argument name and what it does to a DAG.
static int check_dag_list(const SkyoptSession *s, const int32_t *ids, int n, const char *name,
                          const char *verb, const int32_t *ranges, bool every_dag, int n_blocked,
                          std::vector<char> &listed) {
  const int nd = (int)s->dags.size();
  auto check_range = [&](int d, const int32_t *r) {
    if (r[0] < 0 || r[1] < r[0] || r[1] > n_blocked)
      return fail(SKYOPT_EINVAL, "DAG %d: blocked range [%d, %d) is outside [0, %d]", d, r[0], r[1], n_blocked);
    return 0;
  };
  listed.assign(nd, 0);
  for (int k = 0; k < n; ++k) {
    const int d = ids[k];
    if (d < 0 || d >= nd) return fail(SKYOPT_EINVAL, "%s[%d] = %d is outside [0, %d)", name, k, d, nd);
    if (listed[d]) return fail(SKYOPT_EINVAL, "DAG %d is %s twice", d, verb);
    listed[d] = 1;
    if (!every_dag)
      if (int rc = check_range(d, ranges + 2 * k)) return rc;
  }
  for (int d = 0; every_dag && d < nd; ++d)
    if (int rc = check_range(d, ranges + 2 * d)) return rc;
  return 0;
}

// One re-solve of a session: `blocked` replaces the device's blocked table;
// with `all` every DAG takes [0, n_blocked) and is solved again, else the
// `n_listed` DAGs of `dag_ids` take their `ranges` and only their tasks are
// gathered and only they are solved. The other DAGs keep their
// ranges, candidate tables and results in the session's workspace, and the
// solution copied back is the whole workspace's.
// `launched`: launches the caller made before (counted in `stats`).
static int session_resolve(SkyoptSession *s, const SkyoptBlocked *blocked, int n_blocked, bool all,
                           const int32_t *dag_ids, const int32_t *ranges, int n_listed,
                           SkyoptSolution *sol, SkyoptStats *stats, int launched = 0) {
  SkyoptCatalog *cat = s->lease.cat();
  Ctx *x = s->lease.ctx();
  Plan &P = s->P;
  CU(cudaSetDevice(cat->device));
  cudaStream_t st = x->stream;
  int rc;
  if ((rc = s->d_blocked.reserve(sizeof(SkyoptBlocked) * (size_t)n_blocked, st)) ||
      (rc = s->d_dags.reserve(sizeof(SkyoptDag) * s->dags.size(), st)))
    return rc;
  s->ids.clear();
  if (!all) {
    for (int k = 0; k < n_listed; ++k) {
      SkyoptDag &d = s->dags[dag_ids[k]];
      d.blocked_begin = ranges[2 * k]; d.blocked_end = ranges[2 * k + 1];
      for (int t = d.task_begin; t < d.task_end; ++t) s->ids.push_back(t);
    }
  } else {
    for (SkyoptDag &d : s->dags) { d.blocked_begin = 0; d.blocked_end = n_blocked; }
  }
  const int n_tasks = all ? P.nt : (int)s->ids.size();
  const int n_dags = all ? P.nd : n_listed;
  if (!all) s->ids.insert(s->ids.end(), dag_ids, dag_ids + n_listed);
  if ((rc = s->d_ids.reserve(sizeof(int32_t) * s->ids.size(), st))) return rc;
  Launched L;
  L.total_launches = launched;
  CU(cudaEventRecord(x->ev[0], st));
  if (n_dags) {
    // The copies below read pageable host memory: they are staged before the
    // call returns, and the stream is synchronised further down.
    if (n_blocked) CU(cudaMemcpyAsync(s->d_blocked.get(), blocked, sizeof(SkyoptBlocked) * (size_t)n_blocked, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(s->d_dags.get(), s->dags.data(), sizeof(SkyoptDag) * s->dags.size(), cudaMemcpyHostToDevice, st));
    if (!all) CU(cudaMemcpyAsync(s->d_ids.get(), s->ids.data(), sizeof(int32_t) * s->ids.size(), cudaMemcpyHostToDevice, st));
  }
  P.blocked = s->d_blocked.get<SkyoptBlocked>(); P.dags = s->d_dags.get<SkyoptDag>();
  // nothing is scanned or expanded this time: gather and solve only
  CU(cudaEventRecord(x->ev[3], st));
  if (n_dags) {
    const SolveViews v = solve_views(P);
    const int32_t *task_ids = all ? nullptr : s->d_ids.get<int32_t>();
    const int32_t *solve_ids = all ? nullptr : s->d_ids.get<int32_t>() + n_tasks;
    if (n_tasks) {
      gather_kernel<<<n_tasks, kGatherThreads, 0, st>>>(cat->dev, v.in, v.w, P.task_dag, P.task_n, task_ids);
      CU(cudaGetLastError());
      ++L.total_launches;
    }
    solve_kernel<<<n_dags, kSolveThreads, sizeof(ChainSmem), st>>>(cat->dev, v.in, v.w, v.out, P.task_mv, chain_force_full(), solve_ids);
    CU(cudaGetLastError());
    ++L.total_launches;
  }
  CU(cudaEventRecord(x->ev[4], st));
  L.solve = {3, 4};
  CU(cudaMemcpyAsync(x->hbuf.get(), x->dbuf.get() + P.out_off, P.out_bytes, cudaMemcpyDeviceToHost, st));
  CU(cudaEventRecord(x->ev[5], st));
  CU(cudaStreamSynchronize(st));
  SkyoptProblem pb{};
  pb.dags = s->dags.data(); pb.n_dags = (int)s->dags.size();
  if ((rc = copy_solution(cat, x, P, &pb, sol))) return rc;
  return fill_stats(x, L, stats);
}

int skyopt_session_resolve(SkyoptSession *s, const SkyoptBlocked *blocked, int n_blocked,
                           SkyoptSolution *sol, SkyoptStats *stats) {
  NvtxRange nvtx_("skyopt_session_resolve");
  if (!s || !sol || n_blocked < 0 || (n_blocked > 0 && !blocked)) return fail(SKYOPT_EINVAL, "bad arguments");
  return session_resolve(s, blocked, n_blocked, true, nullptr, nullptr, 0, sol, stats);
}

int skyopt_session_resolve_dags(SkyoptSession *s, const SkyoptBlocked *blocked, int n_blocked,
                                const int32_t *dag_ids, const int32_t *ranges, int n_listed,
                                SkyoptSolution *sol, SkyoptStats *stats) {
  NvtxRange nvtx_("skyopt_session_resolve_dags");
  if (!s || !sol || n_blocked < 0 || (n_blocked > 0 && !blocked)) return fail(SKYOPT_EINVAL, "bad arguments");
  if (n_listed < 0) return fail(SKYOPT_EINVAL, "n_listed is negative (%d)", n_listed);
  if (n_listed > 0 && (!dag_ids || !ranges)) return fail(SKYOPT_EINVAL, "dag_ids or ranges is NULL");
  std::vector<char> listed;
  if (int rc = check_dag_list(s, dag_ids, n_listed, "dag_ids", "listed", ranges, false, n_blocked, listed))
    return rc;
  return session_resolve(s, blocked, n_blocked, false, dag_ids, ranges, n_listed, sol, stats);
}

int skyopt_session_update_dags(SkyoptSession *s, const SkyoptBlocked *blocked, int n_blocked,
                               const int32_t *ranges, const int32_t *forced_ids, int n_forced,
                               const SkyoptReservation *reservations, int n_reservations,
                               const int32_t *reservation_ranges, int n_blocks,
                               const int32_t *slot_pad, int n_slots, int32_t *out_ids,
                               int32_t *out_n_ids, SkyoptSolution *sol, SkyoptStats *stats) {
  NvtxRange nvtx_("skyopt_session_update_dags");
  if (!s || !sol || !ranges || !reservation_ranges || !slot_pad || !out_ids || !out_n_ids ||
      n_blocked < 0 || (n_blocked > 0 && !blocked))
    return fail(SKYOPT_EINVAL, "bad arguments");
  if (n_forced < 0 || (n_forced > 0 && !forced_ids))
    return fail(SKYOPT_EINVAL, "bad forced DAG list (%d)", n_forced);
  SkyoptCatalog *cat = s->lease.cat();
  Plan &P = s->P;
  int rc = validate_reservations(cat, reservations, n_reservations, reservation_ranges, n_blocks);
  if (rc) return rc;
  if (n_slots != P.ns)
    return fail(SKYOPT_EINVAL, "n_slots is %d, the session has %d slots", n_slots, P.ns);
  for (int i = 0; i < n_slots; ++i)
    if (slot_pad[i] < 0 || slot_pad[i] > n_blocks)
      return fail(SKYOPT_EINVAL, "slot %d: reservation block %d out of range", i, slot_pad[i] - 1);
  const int nd = (int)s->dags.size();
  std::vector<char> listed;
  if ((rc = check_dag_list(s, forced_ids, n_forced, "forced_ids", "forced", ranges, true, n_blocked, listed)))
    return rc;
  Ctx *x = s->lease.ctx();
  CU(cudaSetDevice(cat->device));
  cudaStream_t st = x->stream;
  // the tasks of COST DAGs with a slot flagged now or after the update
  std::vector<int32_t> tasks;
  for (const SkyoptDag &D : s->dags) {
    if (!D.minimize_cost) continue;
    for (int t = D.task_begin; t < D.task_end; ++t) {
      for (int sl = s->task_slots[2 * t]; sl < s->task_slots[2 * t + 1]; ++sl)
        if (s->pad[sl] || slot_pad[sl]) { tasks.push_back(t); break; }
    }
  }
  const int nxt = s->cur == 0 ? 1 : 0;
  if ((rc = s->d_resv[nxt].reserve(sizeof(SkyoptReservation) * (size_t)n_reservations, st)) ||
      (rc = s->d_resv_off[nxt].reserve(sizeof(int32_t) * ((size_t)n_blocks + 1), st)) ||
      (rc = s->d_tasks.reserve(sizeof(int32_t) * tasks.size(), st)) ||
      (rc = s->d_pad.reserve(sizeof(int32_t) * (size_t)P.ns, st)) ||
      (rc = s->d_marks.reserve(sizeof(int32_t) * (size_t)nd, st)))
    return rc;
  SkyoptReservation *d_resv = s->d_resv[nxt].get<SkyoptReservation>();
  int32_t *d_resv_off = s->d_resv_off[nxt].get<int32_t>(), *d_marks = s->d_marks.get<int32_t>();
  int launched = 0;
  s->marks.assign(nd, 0);
  // The copies read pageable host memory: they are staged before the call
  // returns, and the stream is synchronised below.
  if (n_reservations)
    CU(cudaMemcpyAsync(d_resv, reservations, sizeof(SkyoptReservation) * (size_t)n_reservations,
                       cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(d_resv_off, reservation_ranges, sizeof(int32_t) * ((size_t)n_blocks + 1),
                     cudaMemcpyHostToDevice, st));
  if (!tasks.empty()) {
    CU(cudaMemcpyAsync(s->d_pad.get(), slot_pad, sizeof(int32_t) * (size_t)P.ns, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(s->d_tasks.get(), tasks.data(), sizeof(int32_t) * tasks.size(), cudaMemcpyHostToDevice, st));
    CU(cudaMemsetAsync(d_marks, 0, sizeof(int32_t) * (size_t)nd, st));
    const SolveViews v = solve_views(P);
    reprice_kernel<<<(int)tasks.size(), kRepriceThreads, 0, st>>>(
        v.in, d_resv, d_resv_off, s->d_pad.get<int32_t>(), P.slots, s->d_tasks.get<int32_t>(), P.task_dag, d_marks);
    CU(cudaGetLastError());
    ++launched;
    // the one device-to-host copy of an update before the re-solve: which
    // DAGs the new table re-priced, for the host to list them
    CU(cudaMemcpyAsync(s->marks.data(), d_marks, sizeof(int32_t) * (size_t)nd,
                       cudaMemcpyDeviceToHost, st));
  }
  CU(cudaStreamSynchronize(st));
  // the incoming table is the current one from here on
  s->cur = nxt;
  P.resv = d_resv;
  P.resv_off = d_resv_off;
  s->pad.assign(slot_pad, slot_pad + n_slots);
  // every DAG takes its range of the new blocked table: a re-priced DAG is
  // gathered again and must not read the previous call's entries
  for (int d = 0; d < nd; ++d) {
    s->dags[d].blocked_begin = ranges[2 * d];
    s->dags[d].blocked_end = ranges[2 * d + 1];
  }
  std::vector<int32_t> ids, spans;
  for (int d = 0; d < nd; ++d) {
    if (!listed[d] && !s->marks[d]) continue;
    ids.push_back(d);
    spans.push_back(ranges[2 * d]);
    spans.push_back(ranges[2 * d + 1]);
  }
  std::copy(ids.begin(), ids.end(), out_ids);
  *out_n_ids = (int32_t)ids.size();
  return session_resolve(s, blocked, n_blocked, false, ids.data(), spans.data(), (int)ids.size(),
                         sol, stats, launched);
}

void skyopt_session_close(SkyoptSession *s) {
  if (!s) return;
  cudaSetDevice(s->lease.cat()->device);
  cudaStreamSynchronize(s->lease->stream);
  delete s;
}

int skyopt_solve_tables(SkyoptCatalog *cat, const double *values, const int32_t *clouds,
                        const int64_t *task_offsets, const SkyoptTask *tasks, int n_tasks,
                        const int32_t *parents, int n_parents, const double *tariffs,
                        int n_tariffs, const SkyoptDag *dags, int n_dags,
                        int32_t *chosen_index, SkyoptDagResult *results) {
  NvtxRange nvtx_("skyopt_solve_tables");
  if (!cat || !values || !clouds || !task_offsets || !tasks || !dags || !chosen_index || !results ||
      n_tasks <= 0 || n_dags <= 0)
    return fail(SKYOPT_EINVAL, "bad arguments");
  const int C = cat->dev.n_clouds;
  SkyoptProblem pb{};
  pb.tasks = tasks; pb.n_tasks = n_tasks; pb.parents = parents; pb.n_parents = n_parents;
  pb.tariffs = tariffs; pb.n_tariffs = n_tariffs; pb.dags = dags; pb.n_dags = n_dags;
  // reuse the structural checks (slot ranges are irrelevant here)
  std::vector<SkyoptTask> tk(tasks, tasks + n_tasks);
  for (auto &t : tk) { t.slot_begin = 0; t.slot_end = 0; }
  pb.tasks = tk.data();
  int rc = validate_problem(cat, &pb);
  if (rc) return rc;
  for (int d = 0; d < n_dags; ++d)
    if (dags[d].is_chain == SKYOPT_DAG_SAME_INFRA)
      return fail(SKYOPT_EINVAL, "dag %d: a job group needs regions; these tables have none", d);
  const int64_t total = task_offsets[n_tasks];
  if (task_offsets[0] != 0 || total < 0) return fail(SKYOPT_EINVAL, "bad task_offsets");
  for (int t = 0; t < n_tasks; ++t)
    if (task_offsets[t + 1] < task_offsets[t]) return fail(SKYOPT_EINVAL, "bad task_offsets");
  for (int64_t i = 0; i < total; ++i)
    if (clouds[i] < 0 || clouds[i] >= C) return fail(SKYOPT_EINVAL, "candidate %lld: bad cloud", (long long)i);
  Lease x;
  if ((rc = x.open(cat))) return rc;
  cudaStream_t st = x->stream;
  TablePlan T{total, n_tasks, n_parents, n_tariffs, n_dags, C};
  if ((rc = carve_in(x->dbuf, st, [&](Carver &c) { carve_tables(T, c); }))) return rc;
  std::vector<int32_t> counts(n_tasks);
  for (int t = 0; t < n_tasks; ++t) counts[t] = (int32_t)(task_offsets[t + 1] - task_offsets[t]);
  CU(cudaMemcpyAsync(T.values, values, sizeof(double) * total, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(T.clouds, clouds, sizeof(int32_t) * total, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(T.task_off, task_offsets, sizeof(int64_t) * (n_tasks + 1), cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(T.tasks, tk.data(), sizeof(SkyoptTask) * n_tasks, cudaMemcpyHostToDevice, st));
  if (n_parents) CU(cudaMemcpyAsync(T.parents, parents, sizeof(int32_t) * n_parents, cudaMemcpyHostToDevice, st));
  if (n_tariffs) CU(cudaMemcpyAsync(T.tariffs, tariffs, sizeof(double) * n_tariffs, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(T.dags, dags, sizeof(SkyoptDag) * n_dags, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(T.task_n, counts.data(), sizeof(int32_t) * n_tasks, cudaMemcpyHostToDevice, st));
  SolveIn in{nullptr, T.tasks, T.parents, T.tariffs, nullptr, T.dags, nullptr, T.task_off, ExpandOut{}, 1, nullptr, nullptr};
  SolveWork w{nullptr, nullptr, T.clouds, nullptr, T.values, T.dp, T.back};
  SolveOut out{nullptr, T.chosen_index, T.task_n, T.results};
  solve_kernel<<<n_dags, kSolveThreads, sizeof(ChainSmem), st>>>(cat->dev, in, w, out, T.task_mv, chain_force_full(), nullptr);
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(chosen_index, T.chosen_index, sizeof(int32_t) * n_tasks, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(results, T.results, sizeof(SkyoptDagResult) * n_dags, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  for (int d2 = 0; d2 < n_dags; ++d2)
    if (results[d2].status != 0)
      for (int t = dags[d2].task_begin; t < dags[d2].task_end; ++t) chosen_index[t] = -1;
  return x.finish(0);
}

int skyopt_optimize_timed(SkyoptCatalog *cat, const SkyoptProblem *pb, SkyoptSolution *sol,
                          int iters, int flush_l2, float *iter_ms, float *scan_ms,
                          SkyoptStats *stats) {
  if (!cat || !pb || !sol || iters <= 0 || !iter_ms) return fail(SKYOPT_EINVAL, "bad arguments");
  int rc = validate_problem(cat, pb);
  if (rc) return rc;
  Lease x;
  if ((rc = x.open(cat))) return rc;
  Plan P;
  if ((rc = build_plan(cat, pb, x.ctx(), true, sol->scan != nullptr, P))) return rc;
  cudaStream_t st = x->stream;
  const size_t flush_words = (size_t)(4 * cat->l2_bytes) >> 2;  // four times the L2
  if (flush_l2 && (rc = x->flush.reserve(flush_words * 4, st))) return rc;
  const char *trace_path = getenv("SKYOPT_TRACE");
  const size_t trace_words = (size_t)3 * kTraceBlocks * kTraceSlots;
  if (!trace_path) x->trace = DeviceBuffer();
  else if ((rc = x->trace.reserve(trace_words * 8, st))) return rc;
  unsigned long long *trace = x->trace.get<unsigned long long>();
  CU(cudaEventRecord(x->ev[0], st));
  CU(cudaMemcpyAsync(x->dbuf.get(), x->hbuf.get(), P.in_bytes, cudaMemcpyHostToDevice, st));
  for (int it = 0; it < iters; ++it) {
    if (trace) CU(cudaMemsetAsync(trace, 0, trace_words * 8, st));
    if (flush_l2) {
      flush_kernel<<<cat->sm_count * 8, 256, 0, st>>>(x->flush.get<uint32_t>(), (int64_t)flush_words, (uint32_t)it);
      CU(cudaGetLastError());
    }
    P.fresh_inputs = false;  // the timed region resets the scan results itself
    if ((rc = enqueue_kernels(cat, x.ctx(), P))) return rc;
    CU(cudaStreamSynchronize(st));
    CU(cudaEventElapsedTime(&iter_ms[it], x->ev[1], x->ev[4]));
    if (scan_ms && (rc = elapsed(x.ctx(), P.ran.scan_kernel, &scan_ms[it]))) return rc;
  }
  if (trace) {
    // the last iteration's per-block timeline (tools/trace2.py reads it)
    std::vector<unsigned long long> h(trace_words);
    CU(cudaMemcpy(h.data(), trace, trace_words * 8, cudaMemcpyDeviceToHost));
    // one file per timing loop of the process: <path>, <path>.1, <path>.2, ...
    static int trace_calls = 0;
    std::string path = trace_path;
    if (trace_calls) path += "." + std::to_string(trace_calls);
    ++trace_calls;
    if (FILE *f = fopen(path.c_str(), "wb")) { fwrite(h.data(), 8, h.size(), f); fclose(f); }
  }
  CU(cudaMemcpyAsync(x->hbuf.get(), x->dbuf.get() + P.out_off, P.out_bytes, cudaMemcpyDeviceToHost, st));
  CU(cudaEventRecord(x->ev[5], st));
  CU(cudaStreamSynchronize(st));
  if ((rc = copy_solution(cat, x.ctx(), P, pb, sol))) return rc;
  return x.finish(fill_stats(x.ctx(), P.ran, stats));
}

}  // extern "C"
