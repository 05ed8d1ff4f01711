// skyopt_step.cuh -- the whole optimizer step as ONE persistent cooperative
// kernel: scan2 (filter + argmin) -> grid barrier -> place (expansion, blocked
// filter, cost; block per task) -> chain DP, on a block of its own that starts
// from the minima the task blocks publish after their count pass, or (when the
// grid cannot hold one block per task and per DAG) by the block that finishes a
// DAG's last task. One launch instead of five: on a step of tens of microseconds the
// launch gaps and cold prologues of separate kernels are a large share of the
// time. solve_kernel, at the end, solves DAGs after separate launches with the
// same chain DP.
#pragma once

#include "skyopt_fast.cuh"

namespace skyopt {

// Chain DP (reference sky/optimizer.py:429-487) of one DAG by one block.
//
// The reference walks the chain with, per child candidate c and parent
// candidate p, the sum fl(dp[p] + egress(cloud(p), cloud(c))) and keeps the
// FIRST minimum over p. Egress only depends on the two clouds, so with
//   vmin[t][g] = smallest candidate value of task t in cloud g, idx[t][g] the
//                first candidate holding it (left by the task's place block
//                in the fused step, folded from the tables by solve_kernel),
//   D[t][g]    = fl(vmin[t][g] + B[t][g])     (dp of that candidate),
//   B[t][h]    = min_g fl(D[t-1][g] + e_t(g, h)),  e_t(g, h) = tar_t[g] (g != h), 0 (g == h)
// the recurrence is C wide, and the argmin over g -- ties to the smaller
// candidate index, i.e. the first minimum in candidate order -- IS the
// reference's best parent of every child candidate in cloud h: fl() is
// monotone, so within a cloud no candidate beats the one with the smallest
// value. Same sums, same minima as optimizer.py:456-470, and no candidate is
// ever read. One case needs the full tables: a candidate in FRONT of idx[t][g]
// with a larger value whose sum rounds to the same double would be the
// reference's first minimum. v2[t][g] (the smallest value in front) makes
// that checkable: if fl(fl(v2 + B) + e) == fl(fl(vmin + B) + e) for any cloud
// the block falls back to chain_full() below, which evaluates every candidate.
//
// One task's operands of the lean recurrence (at most four clouds), one row
// per step. Columns C..3 stand for the clouds the general recurrence gives to
// lanes >= C: cloud 0's tariff, no candidate, the largest id.
struct __align__(16) LeanRow {
  double tar[4];   // tariff into cloud g
  double v[4];     // cheapest value in cloud g, +inf when the cloud has none
  int id[4];       // (idx << 5) | g of that candidate
  int np, pad_[3];
};

struct ChainSmem {
  LeanRow lean[kFastTasks];
  double tar[kFastTasks][SKYOPT_MAX_CLOUDS];
  unsigned long long mv[kFastTasks][SKYOPT_MAX_CLOUDS];  // price_key(vmin)
  unsigned long long v2[kFastTasks][SKYOPT_MAX_CLOUDS];  // price_key(v2)
  int mi[kFastTasks][SKYOPT_MAX_CLOUDS];                 // (idx << 5) | cloud
  double B[kFastTasks][SKYOPT_MAX_CLOUDS];
  long long toff[kFastTasks];
  int bk[kFastTasks + 1][SKYOPT_MAX_CLOUDS];  // best parent (idx << 5 | cloud) by child task, child cloud
  int tn[kFastTasks], np[kFastTasks], src[kFastTasks], choice[kFastTasks];
  double obj;
  int first_empty, hazard;
};
// the lean recurrence reads and writes these rows as 16-byte vectors
static_assert(offsetof(ChainSmem, lean) % 16 == 0 && sizeof(LeanRow) % 16 == 0, "LeanRow alignment");
static_assert(offsetof(ChainSmem, B) % 16 == 0 && sizeof(ChainSmem::B[0]) % 16 == 0, "B row alignment");
static_assert(offsetof(ChainSmem, bk) % 16 == 0 && sizeof(ChainSmem::bk[0]) % 16 == 0, "bk row alignment");

__device__ __forceinline__ void step_mark(unsigned long long *trace, int slot) {
  if (trace && threadIdx.x == 0 && blockIdx.x < kTraceBlocks)
    trace[((size_t)2 * kTraceBlocks + blockIdx.x) * kTraceSlots + slot] = global_ns();
}

// (price key, id) pairs in lexicographic order, branch-free
constexpr unsigned long long kKeyInf = 0xFFF0000000000000ull;  // price_key(+inf)
__device__ __forceinline__ bool key_less(unsigned long long ak, int ai, unsigned long long bk, int bi) {
  return (ak < bk) | ((ak == bk) & (ai < bi));
}

// The full evaluation: winners from every candidate's own sum, candidates read
// from the task tables in global memory. Only runs after a hazard (see above),
// so it is written for size, not speed.
template <int kThreads>
__device__ __noinline__ void chain_full(ChainSmem &M, const SolveWork &w, int T, int C, int Cp) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const double kInf = __longlong_as_double(0x7FF0000000000000ll);
  const int parts = 32 / Cp;
  const int h = lane % Cp, part = lane / Cp;
#pragma unroll 1
  for (int lt = warp; lt < T; lt += kThreads / 32) {
    const bool sink = lt == T - 1;
    const int n = M.tn[lt];
    const long long toff = M.toff[lt];
    double bv = kInf; int bi = 0x7FFFFFFF;
    const bool wanted = h < C && (sink ? h == 0 : M.mv[lt + 1][h] != kKeyNone);
    if (wanted) {
#pragma unroll 1
      for (int p = part; p < n; p += parts) {
        const int cp = __ldcg(w.tc_cloud + toff + p) & (SKYOPT_MAX_CLOUDS - 1);
        const double dpp = __dadd_rn(__ldcg(w.tc_value + toff + p), M.B[lt][cp]);
        const double e = (!sink && cp != h) ? M.tar[lt + 1][cp] : 0.0;
        const double sum = sink ? dpp : __dadd_rn(dpp, e);
        if (sum < bv) { bv = sum; bi = p; }
      }
    }
#pragma unroll 1
    for (int o = Cp; o < 32; o <<= 1) {
      const double ov = __shfl_xor_sync(0xFFFFFFFFu, bv, o);
      const int oi = __shfl_xor_sync(0xFFFFFFFFu, bi, o);
      lexmin(bv, bi, ov, oi);
    }
    if (part == 0 && h < C && (!sink || h == 0)) {
      int cl = 0;
      if (bi != 0x7FFFFFFF && bi < n) cl = __ldcg(w.tc_cloud + toff + bi) & (SKYOPT_MAX_CLOUDS - 1);
      M.bk[lt + 1][h] = (int)(((unsigned)bi << 5) | (unsigned)cl);
      if (sink) M.obj = bv;
    }
  }
}

// The recurrence for any number of clouds and any sign of the values: price
// keys (a total order on doubles), butterfly minima for many clouds.
// `kThreads` only gives each kernel its own copy: with a single caller the
// compiler resolves M's shared-memory address inside it rather than taking
// it as a generic pointer.
template <int kThreads>
__device__ __noinline__ void recurrence_general(ChainSmem &M, int T, int C, int Cp, bool &hz, double &bv, int &bi) {
  const int lane = threadIdx.x & 31;
  const double kInf = __longlong_as_double(0x7FF0000000000000ll);
  const int h = lane < C ? lane : 0;
  const bool live = lane < C;
  double dprev = 0.0, hprev = 0.0;   // D[t-1][lane], fl(v2[t-1][lane] + B[t-1][lane])
  int myid = 0x7FFFFFFF;
  bool has2 = false;
  // the next task's operands are fetched one step ahead of the dependent chain
  double tar_n = M.tar[0][h];
  unsigned long long mk_n = M.mv[0][h], v2_n = M.v2[0][h];
  int mi_n = M.mi[0][h], np_n = M.np[0];
#pragma unroll 1
  for (int lt = 0; lt < T; ++lt) {
    const double tar = tar_n;
    const unsigned long long mk = mk_n, v2k = v2_n;
    const int mi = mi_n, np = np_n;
    if (lt + 1 < T) {
      tar_n = M.tar[lt + 1][h]; mk_n = M.mv[lt + 1][h]; v2_n = M.v2[lt + 1][h];
      mi_n = M.mi[lt + 1][h]; np_n = M.np[lt + 1];
    }
    double b;
    if (np == 0) {
      // dummy source: 0 + egress from the inputs' cloud. The addition turns
      // a -0.0 tariff into +0.0, as in the reference; then no D or B below is
      // ever -0.0, so price keys order equal sums as its '<' does.
      b = __dadd_rn(0.0, tar);
    } else {
      const double mine = live ? __dadd_rn(dprev, tar) : kInf;
      // a candidate in front of the cheapest one whose sum rounds the same
      if (live && has2 && dprev < kInf && (hprev == dprev || __dadd_rn(hprev, tar) == mine)) hz = true;
      // The minima are taken on price keys: a total order on doubles as
      // 64-bit integers (equal doubles <=> equal keys for the non-negative
      // sums here). An fp64 compare-and-select costs four times the latency
      // of the integer one, and this loop is nothing but dependent compares.
      const unsigned long long kd = price_key(dprev);
      const unsigned long long km = price_key(mine);
      const int idm = live ? myid : 0x7FFFFFFF;
      unsigned long long bkey = kd;   // own cloud: egress 0
      int bid = myid;
      if (Cp <= 8) {
        // few clouds: every lane reads every cloud's sum (independent
        // shuffles) and keeps a running first minimum -- a third of the
        // instructions of the butterfly below, and one warp's time here is
        // its dependent-instruction count
#pragma unroll 4
        for (int g = 0; g < C; ++g) {
          const unsigned long long kg = __shfl_sync(0xFFFFFFFFu, km, g);
          const int ig = __shfl_sync(0xFFFFFFFFu, idm, g);
          const bool take = (g != lane) & key_less(kg, ig, bkey, bid);
          bkey = take ? kg : bkey;
          bid = take ? ig : bid;
        }
      } else {
        // smallest and second smallest sum (with their ids) by a butterfly;
        // a lane whose own sum is the smallest takes the second
        unsigned long long k1 = km, k2 = kKeyInf;
        int i1 = idm, i2 = 0x7FFFFFFF;
#pragma unroll 1
        for (int o = 1; o < Cp; o <<= 1) {
          const unsigned long long p1 = __shfl_xor_sync(0xFFFFFFFFu, k1, o);
          const int q1 = __shfl_xor_sync(0xFFFFFFFFu, i1, o);
          const unsigned long long p2 = __shfl_xor_sync(0xFFFFFFFFu, k2, o);
          const int q2 = __shfl_xor_sync(0xFFFFFFFFu, i2, o);
          const bool pl = key_less(p1, q1, k1, i1);
          const unsigned long long lo = pl ? p1 : k1, hi = pl ? k1 : p1;
          const int loi = pl ? q1 : i1, hii = pl ? i1 : q1;
          const bool sl = key_less(p2, q2, k2, i2);
          const unsigned long long s2 = sl ? p2 : k2;
          const int s2i = sl ? q2 : i2;
          const bool tl = key_less(s2, s2i, hi, hii);
          k1 = lo; i1 = loi;
          k2 = tl ? s2 : hi; i2 = tl ? s2i : hii;
        }
        const bool own = i1 == myid;   // ids are distinct: (candidate index, cloud)
        const unsigned long long ok = own ? k2 : k1;
        const int oi = own ? i2 : i1;
        const bool ol = key_less(ok, oi, kd, myid);
        bkey = ol ? ok : kd;
        bid = ol ? oi : myid;
      }
      b = key_price(bkey);
      if (live) M.bk[lt][lane] = bid;
    }
    if (live) M.B[lt][lane] = b;
    dprev = (mk == kKeyNone || !live) ? kInf : __dadd_rn(key_price(mk), b);
    has2 = v2k != kKeyNone;
    hprev = has2 ? __dadd_rn(key_price(v2k), b) : 0.0;
    myid = mi;
  }
  // the sink: egress 0 from every cloud, first minimum of D[T-1][.]
  if (live && has2 && dprev < kInf && hprev == dprev) hz = true;
  bv = live ? dprev : kInf;
  bi = live ? myid : 0x7FFFFFFF;
#pragma unroll 1
  for (int o = 1; o < Cp; o <<= 1) {
    const double ov = __shfl_xor_sync(0xFFFFFFFFu, bv, o);
    const int oi = __shfl_xor_sync(0xFFFFFFFFu, bi, o);
    lexmin(bv, bi, ov, oi);
  }
}

// shared memory by 32-bit address: the loop below must not re-derive the
// shared window of a generic pointer at every access
__device__ __forceinline__ void lds_v2_u64(unsigned a, unsigned long long &x, unsigned long long &y) {
  asm volatile("ld.shared.v2.u64 {%0, %1}, [%2];" : "=l"(x), "=l"(y) : "r"(a));
}
__device__ __forceinline__ void lds_v4_s32(unsigned a, int &x, int &y, int &z, int &w) {
  asm volatile("ld.shared.v4.s32 {%0, %1, %2, %3}, [%4];" : "=r"(x), "=r"(y), "=r"(z), "=r"(w) : "r"(a));
}
__device__ __forceinline__ void sts_v2_u64(unsigned a, unsigned long long x, unsigned long long y) {
  asm volatile("st.shared.v2.u64 [%0], {%1, %2};" ::"r"(a), "l"(x), "l"(y) : "memory");
}
__device__ __forceinline__ void sts_v4_s32(unsigned a, int x, int y, int z, int w) {
  asm volatile("st.shared.v4.s32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
}
// the first of two (key, id) pairs in lexicographic order
__device__ __forceinline__ void lexmin_bits(unsigned long long &k, int &i, unsigned long long ok, int oi) {
  const bool lt = (ok < k) | ((ok == k) & (oi < i));
  k = lt ? ok : k; i = lt ? oi : i;
}
__device__ __forceinline__ unsigned long long dadd_bits(unsigned long long a, unsigned long long b) {
  return (unsigned long long)__double_as_longlong(
      __dadd_rn(__longlong_as_double((long long)a), __longlong_as_double((long long)b)));
}

// One LeanRow, the first CP columns (64-bit words as bit patterns): what a
// step needs first (tariffs, parent count), then what it needs last.
template <int CP>
struct LeanHead {
  unsigned long long tar[CP];
  int np;
};
template <int CP>
struct LeanTail {
  unsigned long long v[CP];
  int id[CP];
};
template <int CP>
__device__ __forceinline__ LeanHead<CP> lean_head(unsigned a) {
  LeanHead<CP> r;
  int pad;
  if constexpr (CP == 4) {
    lds_v2_u64(a, r.tar[0], r.tar[1]); lds_v2_u64(a + 16, r.tar[2], r.tar[3]);
  } else if constexpr (CP == 2) {
    lds_v2_u64(a, r.tar[0], r.tar[1]);
  } else {
    unsigned long long x;
    lds_v2_u64(a, r.tar[0], x);
  }
  lds_v4_s32(a + 80, r.np, pad, pad, pad);
  return r;
}
template <int CP>
__device__ __forceinline__ LeanTail<CP> lean_tail(unsigned a) {
  LeanTail<CP> r;
  int pad;
  if constexpr (CP == 4) {
    lds_v2_u64(a + 32, r.v[0], r.v[1]); lds_v2_u64(a + 48, r.v[2], r.v[3]);
    lds_v4_s32(a + 64, r.id[0], r.id[1], r.id[2], r.id[3]);
  } else if constexpr (CP == 2) {
    lds_v2_u64(a + 32, r.v[0], r.v[1]);
    lds_v4_s32(a + 64, r.id[0], r.id[1], pad, pad);
  } else {
    unsigned long long x;
    lds_v2_u64(a + 32, r.v[0], x);
    lds_v4_s32(a + 64, r.id[0], pad, pad, pad);
  }
  return r;
}

// The recurrence for at most four clouds and non-negative values (every real
// request), kept in registers: every lane holds D[t-1][g] and its id for all
// g and computes every cloud's B[t][.] itself, so no lane waits on another.
// One step is a few sums and a small minimum; nothing in it communicates or
// branches.
//   B[t][h] = first minimum of {(D[t-1][h], id_h)} and {(fl(D[t-1][g] + tar[g]), id_g), g != h}
// under (key, id) order.
//
// The hazard test is not in this loop: it only needs D[t-1], v2[t-1] and
// tar[t], all recomputed from the stored B rows by lean_hazard() below.
// Lane 0 stores the B and bk rows; every lane ends with the sink's first
// minimum (bv, bi).
template <int CP>
__device__ __forceinline__ void lean_recurrence(ChainSmem &M, int T, double &bv, int &bi) {
  constexpr unsigned kRow = sizeof(LeanRow), kRowB = SKYOPT_MAX_CLOUDS * 8, kRowK = SKYOPT_MAX_CLOUDS * 4;
  const bool store = (threadIdx.x & 31) == 0;
  unsigned a = (unsigned)__cvta_generic_to_shared(&M.lean[0]);
  const unsigned a_last = (unsigned)__cvta_generic_to_shared(&M.lean[T - 1]);
  unsigned a_B = (unsigned)__cvta_generic_to_shared(&M.B[0][0]);
  unsigned a_bk = (unsigned)__cvta_generic_to_shared(&M.bk[0][0]);
  unsigned long long d[CP];   // bits of D[t-1][g]
  int id[CP];
#pragma unroll
  for (int g = 0; g < CP; ++g) { d[g] = 0; id[g] = 0x7FFFFFFF; }
  LeanHead<CP> nx = lean_head<CP>(a);
#pragma unroll 1
  for (int lt = 0; lt < T; ++lt) {
    const LeanHead<CP> r = nx;
    // values and ids are only wanted at the end of the step, the next step's
    // tariffs at its start (the last row again on the last step: no branch)
    const LeanTail<CP> q = lean_tail<CP>(a);
    a = min(a + kRow, a_last);
    nx = lean_head<CP>(a);
    unsigned long long b[CP]; int bi_[CP];
    unsigned long long k[CP];
#pragma unroll
    for (int g = 0; g < CP; ++g) k[g] = dadd_bits(d[g], r.tar[g]);
    if constexpr (CP == 1) {
      b[0] = d[0]; bi_[0] = id[0];
    } else if constexpr (CP == 2) {
      b[0] = d[0]; bi_[0] = id[0]; lexmin_bits(b[0], bi_[0], k[1], id[1]);
      b[1] = k[0]; bi_[1] = id[0]; lexmin_bits(b[1], bi_[1], d[1], id[1]);
    } else {
      // with tar >= 0, fl(D[h] + tar[h]) >= D[h] under the same id, so the
      // set may take g == h too: one minimum over all g serves every h, and
      // B[t][h] is that against D[t-1][h] (fewer instructions than a
      // minimum per h without its own cloud, and faster on the H100)
      unsigned long long m = k[0], m2 = k[2];
      int mi = id[0], mi2 = id[2];
      lexmin_bits(m, mi, k[1], id[1]);
      lexmin_bits(m2, mi2, k[3], id[3]);
      lexmin_bits(m, mi, m2, mi2);
#pragma unroll
      for (int g = 0; g < CP; ++g) { b[g] = d[g]; bi_[g] = id[g]; lexmin_bits(b[g], bi_[g], m, mi); }
    }
    // a task without parents: 0 + egress from the inputs' cloud
#pragma unroll
    for (int g = 0; g < CP; ++g) b[g] = r.np == 0 ? r.tar[g] : b[g];
    if (store) {
      if constexpr (CP == 4) {
        sts_v2_u64(a_B, b[0], b[1]); sts_v2_u64(a_B + 16, b[2], b[3]);
        sts_v4_s32(a_bk, bi_[0], bi_[1], bi_[2], bi_[3]);
      } else if constexpr (CP == 2) {
        sts_v2_u64(a_B, b[0], b[1]);
        asm volatile("st.shared.v2.s32 [%0], {%1, %2};" ::"r"(a_bk), "r"(bi_[0]), "r"(bi_[1]) : "memory");
      } else {
        asm volatile("st.shared.u64 [%0], %1;" ::"r"(a_B), "l"(b[0]) : "memory");
        asm volatile("st.shared.s32 [%0], %1;" ::"r"(a_bk), "r"(bi_[0]) : "memory");
      }
    }
    a_B += kRowB; a_bk += kRowK;
#pragma unroll
    for (int g = 0; g < CP; ++g) { d[g] = dadd_bits(q.v[g], b[g]); id[g] = q.id[g]; }
  }
  // the sink: egress 0 from every cloud, first minimum of D[T-1][.]
  unsigned long long k = d[0]; int i = id[0];
#pragma unroll
  for (int g = 1; g < CP; ++g) lexmin_bits(k, i, d[g], id[g]);
  bv = __longlong_as_double((long long)k);
  bi = i;
}

// The lean recurrence's hazard test, after it (same predicate as
// recurrence_general's, from the same sums): thread per (step, live cloud).
// Step lt >= 1 with parents looks at D[lt-1][g] and fl(v2[lt-1][g] + B[lt-1][g]);
// lt == T is the sink. Returns whether this thread found one.
template <int kThreads>
__device__ __forceinline__ bool lean_hazard(const ChainSmem &M, int T, int C) {
  constexpr unsigned long long kInfBits = 0x7FF0000000000000ull;
  constexpr unsigned long long kTop = 0x8000000000000000ull;
  bool hz = false;
#pragma unroll 1
  for (int i = threadIdx.x; i < T * C; i += kThreads) {
    const int lt = i / C + 1, g = i % C;
    const unsigned long long mk = M.mv[lt - 1][g], v2k = M.v2[lt - 1][g];
    if (mk == kKeyNone || v2k == kKeyNone) continue;   // D infinite / nothing in front
    const unsigned long long b = (unsigned long long)__double_as_longlong(M.B[lt - 1][g]);
    const unsigned long long d = dadd_bits(mk ^ kTop, b), h2 = dadd_bits(v2k ^ kTop, b);
    if (d >= kInfBits) continue;
    if (lt == T) {
      hz |= h2 == d;
    } else if (M.np[lt] != 0) {
      const unsigned long long tar = (unsigned long long)__double_as_longlong(M.tar[lt][g]);
      hz |= (h2 == d) | (dadd_bits(h2, tar) == dadd_bits(d, tar));
    }
  }
  return hz;
}

__device__ __forceinline__ unsigned int ld_acquire_u32(const unsigned int *p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// A DAG's hand-off word (StepArgs::dag_done): tasks whose minima are published
// in the low half, tasks whose candidate tables are written in the high half.
constexpr int kMinsDone = 1, kTablesDone = 1 << 16;
// one thread waits until the half at `shift` counts all T tasks (the block
// then meets it at a barrier)
__device__ __forceinline__ void poll_hand(const int32_t *hand, int shift, int T) {
  while ((int)((ld_acquire_u32(reinterpret_cast<const unsigned int *>(hand)) >> shift) & 0xFFFFu) < T)
    __nanosleep(32);
}
// every task of the DAG has written its tables; nothing else of this launch
// adds to the word, so it is left at zero for the next one
__device__ __forceinline__ void poll_tables(int32_t *hand, int T) {
  poll_hand(hand, 16, T);
  *hand = 0;
}

// `hand`: null when every task's minima (task_mv) and candidate table are
// written; else the DAG's hand-off word, and the chain waits on it -- first
// for the minima, and for the candidate tables only where it reads them.
// `kThreads`: the block size.
template <int kThreads>
__device__ __forceinline__ void chain_body(const CatDev &cat, const SolveIn &in, const SolveWork &w,
                                           const SolveOut &out, const TaskMin *task_mv,
                                           int dag, int force_full, unsigned char *smem,
                                           int32_t *hand) {
  ChainSmem &M = *reinterpret_cast<ChainSmem *>(smem);
  const SkyoptDag D = in.dags[dag];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int C = cat.n_clouds;
  const int T = D.task_end - D.task_begin;
  step_mark(out.trace, 0);
  // ---- what does not depend on the placement: records and tariffs
  if (tid == 0) { M.first_empty = 0x7FFFFFFF; M.hazard = force_full & 1; }
  int signed_values = (force_full & 2) ? 1 : 0;  // a negative value or tariff anywhere in the DAG
  if (tid < T) {
    const int t = D.task_begin + tid;
    const SkyoptTask TK = in.tasks[t];
    M.toff[tid] = in.task_off[t];
    M.np[tid] = TK.n_parents;
    M.src[tid] = TK.n_parents ? TK.edge_tariff_begin : TK.src_tariff_begin;
  }
  __syncthreads();
#pragma unroll 1
  for (int i = tid; i < T * C; i += kThreads) {
    const int lt = i / C, cc = i % C;
    const double tv = M.src[lt] >= 0 ? in.tariffs[M.src[lt] + cc] : 0.0;
    M.tar[lt][cc] = tv;
    if (__double_as_longlong(tv) < 0 || tv != tv) signed_values = 1;
  }
  if (hand && tid == 0) poll_hand(hand, 0, T);
  __syncthreads();  // (also: the tariffs are in M.tar)
  if (hand) step_mark(out.trace, 2);
  // ---- the minima, left by the tasks' place blocks
  if (tid < T) {
    const int n = __ldcg(out.task_n + D.task_begin + tid);
    M.tn[tid] = n;
    if (n == 0) atomicMin(&M.first_empty, tid);
  }
  const double kInf = __longlong_as_double(0x7FF0000000000000ll);
#pragma unroll 1
  for (int i = tid; i < T * C; i += kThreads) {
    const int lt = i / C, cc = i % C;
    // the cheapest candidate of (task, cloud)
    const ulonglong2 *pm = reinterpret_cast<const ulonglong2 *>(task_mv + (int64_t)(D.task_begin + lt) * C + cc);
    const ulonglong2 m0 = __ldcg(pm), m1 = __ldcg(pm + 1);
    const int id = (int)(((unsigned)m1.x << 5) | (unsigned)cc);
    M.mv[lt][cc] = m0.x;
    M.v2[lt][cc] = m0.y;
    // price keys of non-negative doubles have the top bit set
    if (!(m0.x >> 63) || !(m0.y >> 63)) signed_values = 1;
    M.mi[lt][cc] = id;
    if (C <= 4) {
      // the lean recurrence's row (read only when every value is non-negative)
      LeanRow &R = M.lean[lt];
      const double tv = M.tar[lt][cc];
      R.tar[cc] = tv;
      R.v[cc] = m0.x == kKeyNone ? kInf : key_price(m0.x);
      R.id[cc] = id;
      if (cc == 0) {
        for (int g = C; g < 4; ++g) { R.tar[g] = tv; R.v[g] = kInf; R.id[g] = 0x7FFFFFFF; }
        R.np = M.np[lt];
      }
    }
  }
  const bool lean = __syncthreads_or(signed_values) == 0;
  if (M.first_empty != 0x7FFFFFFF) {
    if (tid == 0) {
      if (hand) poll_tables(hand, T);
      SkyoptDagResult r; r.status = 1; r.task_fail = M.first_empty;
      r.objective = __longlong_as_double(0x7FF8000000000000ll);
      out.dag[dag] = r;
    }
    return;
  }
  step_mark(out.trace, 1);
  const long long c_start = clock64();
  int Cp = 1;
  while (Cp < C) Cp <<= 1;
  if (warp == 0) {
    bool hz = false;
    double bv; int bi;
    if (lean && Cp <= 4) {
      if (Cp == 4) lean_recurrence<4>(M, T, bv, bi);
      else if (Cp == 2) lean_recurrence<2>(M, T, bv, bi);
      else lean_recurrence<1>(M, T, bv, bi);
    } else {
      recurrence_general<kThreads>(M, T, C, Cp, hz, bv, bi);
    }
    const bool any_hz = __any_sync(0xFFFFFFFFu, hz);
    if (lane == 0) {
      M.bk[T][0] = bi; M.obj = bv;
      if (any_hz) M.hazard = 1;
      if (out.trace && blockIdx.x < kTraceBlocks)
        out.trace[((size_t)2 * kTraceBlocks + blockIdx.x) * kTraceSlots + 8] = (unsigned long long)(clock64() - c_start);
    }
  }
  __syncthreads();
  // the lean recurrence's hazard test, from the B rows it stored
  const bool hazard = __syncthreads_or(lean && Cp <= 4 && lean_hazard<kThreads>(M, T, C)) || M.hazard;
  step_mark(out.trace, 3);
  // chain_full and the chosen records read the candidate tables
  if (hazard) {
    if (hand) {
      if (tid == 0) poll_tables(hand, T);
      __syncthreads();
      step_mark(out.trace, 7);
      hand = nullptr;
    }
    chain_full<kThreads>(M, w, T, C, Cp);
    __syncthreads();
  }
  step_mark(out.trace, 4);
  if (tid == 0) {
    int id = M.bk[T][0];
#pragma unroll 1
    for (int lt = T - 1; lt >= 0; --lt) {
      M.choice[lt] = (int)((unsigned)id >> 5);
      if (lt > 0) id = M.bk[lt][id & (SKYOPT_MAX_CLOUDS - 1)];
    }
    SkyoptDagResult r; r.status = 0; r.task_fail = -1; r.objective = M.obj;
    out.dag[dag] = r;
  } else if (hand && tid == 32) {
    // (another warp, while thread 0 back-tracks)
    poll_tables(hand, T);
    if (out.trace && blockIdx.x < kTraceBlocks)
      out.trace[((size_t)2 * kTraceBlocks + blockIdx.x) * kTraceSlots + 7] = global_ns();
  }
  __syncthreads();
  step_mark(out.trace, 5);
  if (tid < T) {
    const int t = D.task_begin + tid;
    const int ci = M.choice[tid];
    out.chosen_index[t] = ci;
    if (!in.tables_only) {
      const int64_t o = M.toff[tid] + ci;
      const int64_t ref = __ldcg(w.tc_ref + o);
      const int s = __ldcg(w.tc_slot + o);
      SkyoptCandidate c;
      c.slot = s;
      c.inst_id = __ldcg(in.ex.slot_inst + s);
      c.region_id = __ldcg(in.ex.cand_region + ref);
      c.zone_id = __ldcg(in.ex.cand_zone + ref);
      c.hourly = __ldcg(w.tc_hourly + o);
      c.value = __ldcg(w.tc_value + o);
      out.chosen[t] = c;
    }
  }
  step_mark(out.trace, 6);
}

struct StepArgs {
  Scan2Args scan;
  PlaceArgs place;
  SolveOut out;
  const int32_t *task_dag;
  int n_tasks, n_queries;
  const char *in_base;    // the uploaded input region (descriptors), prefetched into L2
  int64_t in_lines;
  int do_solve;           // every DAG is a chain of <= kFastTasks tasks
  // with do_solve: DAG d's chain DP runs on block n_tasks + d, which places
  // nothing and starts from the minima as the tasks publish them (needs
  // n_tasks + n_dags <= gridDim.x); else on the block that places its last task
  int chain_blocks;
  int n_dags;
  int force_full;         // test knobs: bit 0 chain_full() on every DAG (SKYOPT_EXP=8), bit 1 the general recurrence (SKYOPT_EXP=16)
  int32_t *dag_done;      // [n_dags] hand-off words, kMinsDone / kTablesDone (zero between launches)
  unsigned int *sync;     // arrivals at the grid barrier, counted across launches
  unsigned int sync_target;  // ... and the count that completes this launch's barrier
  // the other copy of the scan results: re-armed here for the next launch of a
  // device-resident loop, by blocks that have passed the barrier
  uint32_t *next_best_rank, *next_any1;
  unsigned int *next_group_ready;
};

__global__ void __launch_bounds__(kScanThreads, kScanBlocksPerSM) step_kernel(const __grid_constant__ StepArgs a) {
  extern __shared__ __align__(128) unsigned char smem_step[];
  __shared__ int s_last;
  __shared__ int s_dag0[2];  // the first task's DAG and its task count (not kept in registers through the loop)
  const int tid = threadIdx.x;
  if (blockIdx.x == 0 && tid == 0 && a.scan.zero_flag) *a.scan.zero_flag = 0;
  // the problem's descriptors (tens of KB) are wanted in L2 by the later
  // phases: every block touches its share of the lines now
  for (int64_t line = (int64_t)blockIdx.x * kScanThreads + tid; line < a.in_lines;
       line += (int64_t)gridDim.x * kScanThreads)
    asm volatile("prefetch.global.L2 [%0];" ::"l"(a.in_base + line * 128));
  ScanWin win{nullptr, 0};
  if (a.scan.n_pieces) win = scan2_body(a.scan, smem_step);
  // ---- grid barrier: every scan result is published (cooperative launch:
  // all blocks are resident)
  __syncthreads();  // (also: the scan's shared memory is free)
  if (tid == 0) {
    __threadfence();
    atomicAdd(a.sync, 1u);
  }
  // Once arrived, until the barrier opens: what the block's first task needs
  // that no scan result decides (its DAG, its placement's inputs), and, where
  // this block's best lowered a query's, that row's launchable list into L2.
  // Nothing read here is written in this launch.
  const int t0 = blockIdx.x;
  if (t0 < a.n_tasks) {
    if (a.do_solve && tid == 0) {
      const int dag = a.task_dag[t0];
      const SkyoptDag D = a.place.in.dags[dag];
      s_dag0[0] = dag; s_dag0[1] = D.task_end - D.task_begin;
    }
    place_stage(a.place, t0, smem_step, true);
  }
  if (win.rec) {
    const int inst = win.rec->inst, off = win.rec->list_off, n = win.rec->cnt[win.col];
    if (inst >= 0) warm_l2(a.scan.f.exp_ent[win.col] + off, (int64_t)n * (int64_t)sizeof(ExpEnt));
  }
  if (tid == 0) {
    // (the counter only grows: the host passes the total that ends this
    // launch's barrier, so nothing has to be reset on the way out)
    while ((int)(ld_acquire_u32(a.sync) - a.sync_target) < 0) __nanosleep(64);
    __threadfence();
  }
  __syncthreads();
  // ---- re-arm the other copy of the scan results (nobody reads it in this
  // launch): a few stores per block, off the critical path
#pragma unroll 1
  for (int i = blockIdx.x * kScanThreads + tid; i < a.n_queries; i += gridDim.x * kScanThreads) {
    a.next_best_rank[i] = kRankNone; a.next_any1[i] = 0u;
  }
  if (a.scan.group_ready)
#pragma unroll 1
    for (int i = blockIdx.x * kScanThreads + tid; i < a.scan.n_groups; i += gridDim.x * kScanThreads)
      a.next_group_ready[i] = 0u;
  const int n_work = a.n_tasks + (a.chain_blocks ? a.n_dags : 0);
  for (int t = blockIdx.x; t < n_work; t += gridDim.x) {
    int chain = -1;           // the DAG whose chain DP this block runs now
    int32_t *hand = nullptr;  // ... and its hand-off word, when it runs beside the placement
    if (t >= a.n_tasks) {
      // a block that places nothing (chain_blocks: the grid covers every task)
      const int dag = t - a.n_tasks;
      const SkyoptDag D = a.place.in.dags[dag];
      if (D.task_end > D.task_begin) { chain = dag; hand = a.dag_done + dag; }
    } else {
      // which DAG, and how many tasks it has: asked for before the placement,
      // needed right after it (the block's first task: staged above)
      int dag = 0, dag_tasks = 0;
      if (t == t0) {
        if (a.do_solve) { dag = s_dag0[0]; dag_tasks = s_dag0[1]; }
      } else {
        if (a.do_solve) {
          dag = a.task_dag[t];
          const SkyoptDag D = a.place.in.dags[dag];
          dag_tasks = D.task_end - D.task_begin;
        }
        place_stage(a.place, t, smem_step, false);
        __syncthreads();
      }
      place_resolve(a.place, t, smem_step, a.chain_blocks ? a.dag_done + dag : nullptr);
      if (a.do_solve) {
        __syncthreads();  // the task's tables are written
        if (tid == 0) {
          __threadfence();
          const int done = atomicAdd(a.dag_done + dag, kTablesDone);
          s_last = (!a.chain_blocks && (done >> 16) == dag_tasks - 1) ? 1 : 0;
          if (s_last) a.dag_done[dag] = 0;  // ready for the next launch
        }
        __syncthreads();
        if (s_last) chain = dag;
      }
    }
    if (chain >= 0) {
      __threadfence();
      chain_body<kScanThreads>(a.scan.cat, a.place.in, a.place.w, a.out, a.place.task_mv, chain, a.force_full, smem_step, hand);
    }
    __syncthreads();  // shared memory is reused by the next task
  }
}


// ---------------------------------------------------------------------------
// K3: one block per DAG, once its tasks' candidate tables are written.
constexpr int kSolveThreads = 1024;  // 32 warps: the minima fold gives one to each task of a short chain
constexpr int kMaxDagTasks = 16;     // exact search only; chains are unbounded

// What the minima fold of solve_kernel keeps per (task, cloud) while it runs;
// it lives in the chain DP's shared memory, which chain_body fills after it.
struct MinFold {
  unsigned long long vmin[kFastTasks][SKYOPT_MAX_CLOUDS];  // smallest price key
  unsigned long long v2[kFastTasks][SKYOPT_MAX_CLOUDS];    // smallest key in front of idx
  unsigned int idx[kFastTasks][SKYOPT_MAX_CLOUDS];         // first candidate holding vmin
};
static_assert(sizeof(MinFold) <= sizeof(ChainSmem), "MinFold shares the chain DP's shared memory");

// Dynamic shared memory: sizeof(ChainSmem). `task_mv`: [n_tasks][n_clouds]
// TaskMin records, written here for the chains of at most kFastTasks tasks;
// `force_full`: the test knobs of StepArgs::force_full.
__global__ void __launch_bounds__(kSolveThreads)
solve_kernel(CatDev cat, SolveIn in, SolveWork w, SolveOut out, TaskMin *task_mv, int force_full) {
  extern __shared__ __align__(16) unsigned char smem_solve[];
  constexpr int kWarps = kSolveThreads / 32;
  __shared__ int s_fail;
  __shared__ double s_best_val[SKYOPT_MAX_CLOUDS];
  __shared__ int s_best_idx[SKYOPT_MAX_CLOUDS];
  __shared__ double s_tb_val[kMaxDagTasks][SKYOPT_MAX_CLOUDS];
  __shared__ int s_tb_idx[kMaxDagTasks][SKYOPT_MAX_CLOUDS];
  __shared__ int s_opt[kMaxDagTasks][SKYOPT_MAX_CLOUDS];  // cloud options
  __shared__ int s_nopt[kMaxDagTasks];
  __shared__ double s_red_val[kWarps];
  __shared__ long long s_red_idx[kWarps];

  step_mark(out.trace, 0);
  const SkyoptDag D = in.dags[blockIdx.x];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int C = cat.n_clouds;
  const int T = D.task_end - D.task_begin;
  if (D.is_chain && T <= kFastTasks) {
    // ---- Chains of up to kFastTasks tasks: the fused step's chain DP
    // (chain_body), which also reports the first task without a candidate.
    // Its per-(task, cloud) minima are folded from the written tables in
    // three order-free passes: the smallest price key, the first candidate
    // holding it, the smallest key in front of that one. Every warp takes
    // part, kWarps / T of them per task.
    MinFold &F = *reinterpret_cast<MinFold *>(smem_solve);
    for (int i = tid; i < T * C; i += kSolveThreads) {
      F.vmin[i / C][i % C] = kKeyNone; F.v2[i / C][i % C] = kKeyNone; F.idx[i / C][i % C] = 0x7FFFFFFFu;
    }
    const int per_task = kWarps / T, lt = warp / per_task;
    const int64_t toff = lt < T ? in.task_off[D.task_begin + lt] : 0;
    const int n = lt < T ? out.task_n[D.task_begin + lt] : 0;
    __syncthreads();
    auto each = [&](auto f) {
      for (int c = (warp % per_task) * 32 + lane; c < n; c += per_task * 32)
        f(w.tc_cloud[toff + c], (unsigned)c, price_key(w.tc_value[toff + c]));
      __syncthreads();
    };
    each([&](int cl, unsigned c, unsigned long long k) { atomicMin(&F.vmin[lt][cl], k); });
    each([&](int cl, unsigned c, unsigned long long k) { if (k == F.vmin[lt][cl]) atomicMin(&F.idx[lt][cl], c); });
    each([&](int cl, unsigned c, unsigned long long k) { if (c < F.idx[lt][cl]) atomicMin(&F.v2[lt][cl], k); });
    for (int i = tid; i < T * C; i += kSolveThreads) {
      TaskMin m;
      m.vmin = F.vmin[i / C][i % C]; m.v2 = F.v2[i / C][i % C]; m.idx = (int32_t)F.idx[i / C][i % C];
      m.pad_[0] = m.pad_[1] = m.pad_[2] = 0;
      task_mv[(int64_t)D.task_begin * C + i] = m;
    }
    __syncthreads();
    chain_body<kSolveThreads>(cat, in, w, out, task_mv, blockIdx.x, force_full, smem_solve, nullptr);
    return;
  }

  if (tid == 0) s_fail = -1;
  __syncthreads();

  // ---- Phase A ran before this kernel: candidate tables are ready. First
  // task without a candidate (all tasks are checked at once: a serial scan
  // would be one dependent memory round trip per task).
  __shared__ int s_first_empty;
  if (tid == 0) s_first_empty = 0x7FFFFFFF;
  __syncthreads();
  for (int lt = tid; lt < T; lt += kSolveThreads)
    if (out.task_n[D.task_begin + lt] == 0) atomicMin(&s_first_empty, lt);
  __syncthreads();
  if (tid == 0 && s_first_empty != 0x7FFFFFFF) s_fail = s_first_empty;
  __syncthreads();
  if (s_fail >= 0) {
    if (tid == 0) {
      SkyoptDagResult r; r.status = 1; r.task_fail = s_fail;
      r.objective = __longlong_as_double(0x7FF8000000000000ll);
      out.dag[blockIdx.x] = r;
    }
    return;
  }

  const double kInf = __longlong_as_double(0x7FF0000000000000ll);
  step_mark(out.trace, 1);

  if (D.is_chain) {
    // ---- Phase B: dp[c] = value[c] + min_p (dp[p] + egress(p, c)); strict
    // '<' => first minimum in candidate order (optimizer.py:456-470). The
    // egress term depends on the clouds only, so the inner minimum is taken
    // once per child cloud -- same additions, same comparisons, same winner.
    for (int t = D.task_begin; t < D.task_end; ++t) {
      const SkyoptTask TK = in.tasks[t];
      const int64_t toff = in.task_off[t];
      const int n = out.task_n[t];
      if (TK.n_parents == 0) {
        if (tid < C) {
          // parent = dummy source: 0 + egress from the inputs' cloud (the
          // addition makes a -0.0 tariff +0.0, so no dp and no objective is -0.0)
          s_best_val[tid] = __dadd_rn(0.0, TK.src_tariff_begin >= 0 ? in.tariffs[TK.src_tariff_begin + tid] : 0.0);
          s_best_idx[tid] = 0;
        }
      } else {
        const int tp = D.task_begin + in.parents[TK.parent_begin];
        const int64_t poff = in.task_off[tp];
        const int np = out.task_n[tp];
        const double *tar = in.tariffs + TK.edge_tariff_begin;
        for (int cc = warp; cc < C; cc += kWarps) {
          double bv = kInf; int bi = 0x7FFFFFFF;
          for (int p = lane; p < np; p += 32) {
            const int cp = w.tc_cloud[poff + p];
            const double eg = (cp != cc) ? tar[cp] : 0.0;
            lexmin(bv, bi, __dadd_rn(w.dp[poff + p], eg), p);
          }
          for (int o = 16; o; o >>= 1) {
            const double ov = __shfl_xor_sync(0xFFFFFFFFu, bv, o);
            const int oi = __shfl_xor_sync(0xFFFFFFFFu, bi, o);
            lexmin(bv, bi, ov, oi);
          }
          if (lane == 0) { s_best_val[cc] = bv; s_best_idx[cc] = bi; }
        }
      }
      __syncthreads();
      for (int c = tid; c < n; c += kSolveThreads) {
        const int cc = w.tc_cloud[toff + c];
        w.dp[toff + c] = __dadd_rn(w.tc_value[toff + c], s_best_val[cc]);
        w.back[toff + c] = s_best_idx[cc];
      }
      __syncthreads();
    }
    // sink: 0 + min_p dp[p] (egress to the dummy sink is 0)
    {
      const int t = D.task_end - 1;
      const int64_t toff = in.task_off[t];
      const int n = out.task_n[t];
      double bv = kInf; int bi = 0x7FFFFFFF;
      for (int p = tid; p < n; p += kSolveThreads) lexmin(bv, bi, w.dp[toff + p], p);
      for (int o = 16; o; o >>= 1) {
        const double ov = __shfl_xor_sync(0xFFFFFFFFu, bv, o);
        const int oi = __shfl_xor_sync(0xFFFFFFFFu, bi, o);
        lexmin(bv, bi, ov, oi);
      }
      if (lane == 0) { s_red_val[warp] = bv; s_red_idx[warp] = bi; }
      __syncthreads();
      if (tid == 0) {
        for (int k = 1; k < kWarps; ++k) lexmin(bv, bi, s_red_val[k], (int)s_red_idx[k]);
        SkyoptDagResult r; r.status = 0; r.task_fail = -1; r.objective = bv;
        out.dag[blockIdx.x] = r;
        int idx = bi;
        for (int tt = D.task_end - 1; tt >= D.task_begin; --tt) {
          out.chosen_index[tt] = idx;
          idx = w.back[in.task_off[tt] + idx];
        }
      }
    }
  } else {
    // ---- Phase B': exact search replacing the PuLP/CBC ILP
    // (optimizer.py:490-637). Egress depends on (cloud_u, cloud_v) only, so
    // within one cloud the cheapest candidate of a task dominates; what is
    // left is an exhaustive enumeration of cloud assignments.
    if (T > kMaxDagTasks) {
      if (tid == 0) {
        SkyoptDagResult r; r.status = 2; r.task_fail = -1;
        r.objective = __longlong_as_double(0x7FF8000000000000ll);
        out.dag[blockIdx.x] = r;
      }
      return;
    }
    for (int lt = warp; lt < T; lt += kWarps) {
      const int t = D.task_begin + lt;
      const int64_t toff = in.task_off[t];
      const int n = out.task_n[t];
      for (int cc = 0; cc < C; ++cc) {
        double bv = kInf; int bi = 0x7FFFFFFF;
        for (int p = lane; p < n; p += 32)
          if (w.tc_cloud[toff + p] == cc) lexmin(bv, bi, w.tc_value[toff + p], p);
        for (int o = 16; o; o >>= 1) {
          const double ov = __shfl_xor_sync(0xFFFFFFFFu, bv, o);
          const int oi = __shfl_xor_sync(0xFFFFFFFFu, bi, o);
          lexmin(bv, bi, ov, oi);
        }
        if (lane == 0) { s_tb_val[lt][cc] = bv; s_tb_idx[lt][cc] = bi; }
      }
      __syncwarp();
      if (lane == 0) {
        // options ordered by the candidate index of their representative
        int no = 0;
        for (int cc = 0; cc < C; ++cc)
          if (s_tb_idx[lt][cc] != 0x7FFFFFFF) s_opt[lt][no++] = cc;
        for (int a = 1; a < no; ++a) {
          const int v = s_opt[lt][a]; int b2 = a - 1;
          while (b2 >= 0 && s_tb_idx[lt][s_opt[lt][b2]] > s_tb_idx[lt][v]) { s_opt[lt][b2 + 1] = s_opt[lt][b2]; --b2; }
          s_opt[lt][b2 + 1] = v;
        }
        s_nopt[lt] = no;
      }
    }
    __syncthreads();
    long long total = 1;
    bool too_big = false;
    for (int lt = 0; lt < T; ++lt) {
      total *= s_nopt[lt];
      if (total > (1ll << 26)) { too_big = true; break; }  // ~10 ms of one block; beyond: status 2
    }
    if (too_big) {
      if (tid == 0) {
        SkyoptDagResult r; r.status = 2; r.task_fail = -1;
        r.objective = __longlong_as_double(0x7FF8000000000000ll);
        out.dag[blockIdx.x] = r;
      }
      return;
    }
    double bv = kInf; long long bid = 0x7FFFFFFFFFFFFFFFll;
    for (long long id = tid; id < total; id += kSolveThreads) {
      int cl[kMaxDagTasks];
      long long rem = id;
      for (int lt = T - 1; lt >= 0; --lt) {  // task 0 = most significant digit
        const int no = s_nopt[lt];
        cl[lt] = s_opt[lt][(int)(rem % no)];
        rem /= no;
      }
      double obj;
      if (D.minimize_cost) {
        obj = 0.0;
        for (int lt = 0; lt < T; ++lt) obj = __dadd_rn(obj, s_tb_val[lt][cl[lt]]);
        for (int lt = 0; lt < T; ++lt) {
          const SkyoptTask TK = in.tasks[D.task_begin + lt];
          if (TK.n_parents == 0 && TK.src_tariff_begin >= 0)
            obj = __dadd_rn(obj, in.tariffs[TK.src_tariff_begin + cl[lt]]);
          for (int k = 0; k < TK.n_parents; ++k) {
            const int lp = in.parents[TK.parent_begin + k];
            if (cl[lp] != cl[lt])
              obj = __dadd_rn(obj, in.tariffs[TK.edge_tariff_begin + k * C + cl[lp]]);
          }
        }
      } else {
        double fin[kMaxDagTasks];
        obj = 0.0;
        for (int lt = 0; lt < T; ++lt) {
          const SkyoptTask TK = in.tasks[D.task_begin + lt];
          double start = 0.0;
          if (TK.n_parents == 0 && TK.src_tariff_begin >= 0)
            start = fmax(start, in.tariffs[TK.src_tariff_begin + cl[lt]]);
          for (int k = 0; k < TK.n_parents; ++k) {
            const int lp = in.parents[TK.parent_begin + k];
            const double eg = (cl[lp] != cl[lt])
                                  ? in.tariffs[TK.edge_tariff_begin + k * C + cl[lp]] : 0.0;
            start = fmax(start, __dadd_rn(fin[lp], eg));
          }
          fin[lt] = __dadd_rn(s_tb_val[lt][cl[lt]], start);
          // the sink waits for the leaves; the largest finish time of any task
          // is the same only because values and tariffs are >= 0 (a task never
          // finishes after a descendant)
          obj = fmax(obj, fin[lt]);
        }
      }
      if (obj < bv || (obj == bv && id < bid)) { bv = obj; bid = id; }
    }
    for (int o = 16; o; o >>= 1) {
      const double ov = __shfl_xor_sync(0xFFFFFFFFu, bv, o);
      const long long oi = __shfl_xor_sync(0xFFFFFFFFu, bid, o);
      if (ov < bv || (ov == bv && oi < bid)) { bv = ov; bid = oi; }
    }
    if (lane == 0) { s_red_val[warp] = bv; s_red_idx[warp] = bid; }
    __syncthreads();
    if (tid == 0) {
      for (int k = 1; k < kWarps; ++k)
        if (s_red_val[k] < bv || (s_red_val[k] == bv && s_red_idx[k] < bid)) { bv = s_red_val[k]; bid = s_red_idx[k]; }
      SkyoptDagResult r; r.status = 0; r.task_fail = -1; r.objective = bv;
      out.dag[blockIdx.x] = r;
      long long rem = bid;
      for (int lt = T - 1; lt >= 0; --lt) {
        const int no = s_nopt[lt];
        const int cc = s_opt[lt][(int)(rem % no)];
        rem /= no;
        out.chosen_index[D.task_begin + lt] = s_tb_idx[lt][cc];
      }
    }
  }
  __syncthreads();
  step_mark(out.trace, 5);
  if (in.tables_only) return;
  // ---- the plan as candidate records
  for (int lt = tid; lt < T; lt += kSolveThreads) {
    const int t = D.task_begin + lt;
    const int64_t o = in.task_off[t] + out.chosen_index[t];
    const int64_t ref = w.tc_ref[o];
    const int s = w.tc_slot[o];
    SkyoptCandidate c;
    c.slot = s;
    c.inst_id = in.ex.slot_inst[s];
    c.region_id = in.ex.cand_region[ref];
    c.zone_id = in.ex.cand_zone[ref];
    c.hourly = w.tc_hourly[o];
    c.value = w.tc_value[o];
    out.chosen[t] = c;
  }
  step_mark(out.trace, 6);
}

}  // namespace skyopt
