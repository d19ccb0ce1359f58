// DisaggregatedSet sweep (sm_90a): one thread per DisaggregatedSet, the ≤10
// roles of a DS in registers / local arrays.
//
// Follows pkg/controllers/disaggregatedset/{planner.go:61-352, executor.go:
// 199-302,306-398, disaggregatedset_controller.go:95-112,137-186,203-236,
// service_manager.go:57-89,174-189}.  The reference's float64 step arithmetic
// (planner.go:92,103-104,125,139-140) is evaluated in 64-bit integers: for
// non-negative a, b, c with a·b < 2^53 the IEEE quotient a·b/c lies on the same
// side of every integer as the exact one, so int(x), floor(x) and ceil(x) equal
// integer floor / ceil division (DESIGN.md "float vs int"); the CPU oracle keeps
// the float form, so parity tests compare the two formulations.
#include "lwse_device.cuh"
#include "lwse_launch.cuh"

namespace lwse {

constexpr int MAXR = (int)LWSE_DS_MAX_ROLES;

struct RuConfig {
  int ms, mu;
};

__device__ __forceinline__ int batch_size(int ms, int mu) { return ms > 0 ? ms : max(1, mu); }  // :61-66

// floor(a*b/c) and ceil(a*b/c) for a,b >= 0, c > 0
__device__ __forceinline__ int floor_muldiv(int a, int b, int c) { return (int)(((long long)a * b) / c); }
__device__ __forceinline__ int ceil_muldiv(int a, int b, int c) {
  return (int)((((long long)a * b) + c - 1) / c);
}

// planner.go:264-294
__device__ void apply_orphan_prevention(int n, int* next_old, const int* cur_new, const int* initial_old,
                                        const int* target, const RuConfig* cfg) {
  bool any_zero = false, all_zero = true;
  for (int i = 0; i < n; i++) {
    if (initial_old[i] == 0) continue;
    if (next_old[i] == 0)
      any_zero = true;
    else
      all_zero = false;
  }
  if (!any_zero || all_zero) return;
  bool can_all = true;  // canDrainAllToZero :252-262
  for (int i = 0; i < n; i++)
    if (initial_old[i] >= target[i] && cur_new[i] < target[i] - cfg[i].mu) can_all = false;
  if (can_all) {
    for (int i = 0; i < n; i++) next_old[i] = 0;
    return;
  }
  for (int i = 0; i < n; i++)
    if (next_old[i] == 0 && initial_old[i] > 0) next_old[i] = 1;
}

// planner.go:320-352 ComputeNextStep → true when a step exists
__device__ bool compute_next_step(int n, const int* initial_old, const int* cur_old, const int* cur_new,
                                  const int* target, const RuConfig* cfg, int* past, int* new_) {
  bool complete = true;  // :173-180
  for (int i = 0; i < n; i++)
    if (cur_old[i] != 0 || cur_new[i] < target[i]) complete = false;
  if (complete) return false;
  int total_steps = 0;  // :68-78
  for (int i = 0; i < n; i++) {
    const int mx = max(max(initial_old[i], target[i]), 0);
    const int b = batch_size(cfg[i].ms, cfg[i].mu);
    total_steps = max(total_steps, (mx + b - 1) / b);
  }
  if (total_steps == 0) return false;
  {  // correctAbnormalState :151-171
    bool needs = false;
    for (int i = 0; i < n; i++) {
      past[i] = min(initial_old[i], cur_old[i]);
      if (cur_old[i] > past[i]) needs = true;
      new_[i] = cur_new[i];
    }
    if (needs) return true;
  }
  {  // isNewAtTarget :182-189
    bool at = true;
    for (int i = 0; i < n; i++)
      if (cur_new[i] < target[i]) at = false;
    if (at) {
      for (int i = 0; i < n; i++) {
        past[i] = 0;
        new_[i] = cur_new[i];
      }
      return true;
    }
  }
  int next_new[MAXR], min_old[MAXR];
  {  // computeNextNewReplicas :80-113
    int min_idx = total_steps;
    for (int i = 0; i < n; i++) {
      const int idx = target[i] == 0 ? total_steps : floor_muldiv(cur_new[i], total_steps, target[i]);
      min_idx = min(min_idx, idx);
    }
    const int next_idx = min_idx + 1;
    for (int i = 0; i < n; i++) {
      const int computed = min(ceil_muldiv(next_idx, target[i], total_steps), target[i]);
      next_new[i] = max(computed, cur_new[i]);
    }
  }
  for (int i = 0; i < n; i++) {  // computeMinOld :203-211
    min_old[i] = 0;
    if (initial_old[i] >= target[i]) min_old[i] = max(0, target[i] - cfg[i].mu - cur_new[i]);
  }
  {  // tryScaleUp :213-228, canScaleUp :191-201
    bool needs = false, can = true;
    for (int i = 0; i < n; i++) {
      if (next_new[i] > cur_new[i]) needs = true;
      if (target[i] != 0 && cur_old[i] + next_new[i] > target[i] + cfg[i].ms) can = false;
    }
    if (needs && can) {
      for (int i = 0; i < n; i++) {
        past[i] = cur_old[i];
        new_[i] = next_new[i];
      }
      return true;
    }
  }
  {  // tryProportionalDrain :230-250 (computeNextOldReplicas :115-149)
    int next_old[MAXR];
    int max_idx = 0;
    for (int i = 0; i < n; i++) {
      if (initial_old[i] == 0) continue;
      max_idx = max(max_idx, floor_muldiv(initial_old[i] - cur_old[i], total_steps, initial_old[i]));
    }
    const int next_idx = max_idx + 1;
    bool needs = false;
    for (int i = 0; i < n; i++) {
      const int computed = max(0, initial_old[i] - floor_muldiv(next_idx, initial_old[i], total_steps));
      next_old[i] = max(min(computed, cur_old[i]), min_old[i]);
    }
    apply_orphan_prevention(n, next_old, cur_new, initial_old, target, cfg);
    for (int i = 0; i < n; i++)
      if (next_old[i] < cur_old[i]) needs = true;
    if (needs) {
      for (int i = 0; i < n; i++) {
        past[i] = next_old[i];
        new_[i] = cur_new[i];
      }
      return true;
    }
  }
  {  // tryForceDrain :296-318
    int drained[MAXR];
    bool needs = false;
    for (int i = 0; i < n; i++) {
      const int max_old = target[i] + cfg[i].ms - next_new[i];
      drained[i] = max(0, min(cur_old[i], max_old));
      if (initial_old[i] >= target[i]) drained[i] = max(drained[i], max(0, target[i] - cfg[i].mu - next_new[i]));
      if (drained[i] < cur_old[i]) needs = true;
    }
    if (needs) {
      apply_orphan_prevention(n, drained, next_new, initial_old, target, cfg);
      for (int i = 0; i < n; i++) {
        past[i] = drained[i];
        new_[i] = next_new[i];
      }
      return true;
    }
  }
  return false;
}

// The resident DS tick (lwse_ds_resident_tick): t's outputs are this tick's output set; the
// previous tick's results are in the other set (the sweep uses revrole_out as scratch inside
// scaleDownOld, so it cannot be compared in place).
struct DsTickArgs {
  const lwse_ds_out* prev_ds_out;
  const lwse_ds_role_out* prev_role_out;
  const lwse_ds_revrole_out* prev_revrole_out;
  lwse_ds_out* m_ds_out;  // pinned, mapped mirrors of the full output tables
  lwse_ds_role_out* m_role_out;
  lwse_ds_revrole_out* m_revrole_out;
  uint8_t* marks;      // DS rows the tick's scatter patched (cleared here)
  uint32_t* rows;      // pinned, mapped: the changed DS rows
  uint32_t* count;     // device: rows appended so far (reset by the publishing CTA)
  uint32_t* ticket;    // device: CTAs done (reset by the publishing CTA)
  uint32_t* host_words;  // pinned, mapped: [0] changed rows, [1] sequence word
  uint32_t seq;
  uint32_t all;        // first tick after a load: every DS is listed
  // linked tick only (kLinked): the link table and the resident LWS rows it points into
  const lwse_ds_link* links;  // [n_revroles]
  const lwse_lws_rec* lws;    // resident LWS table and the results of the last LWS sweep enqueued
  const lwse_lws_out* lws_out;
  uint32_t n_lws;             // 0: no LWS tables or no results yet (every linked row falls back)
};

// The ready count a linked revision-role row uses (lwse.h, LWSE_TABLE_DS_LINKS): the child's
// lws_out.ready_replicas when the row exists, its link names a row < n_lws, that row still holds the
// same object (uid_hash) and its result went through Status().Update; else the row's own value.
// Counts rows that took the LWS value (took) and linked rows that fell back (fell).  The LWS rows
// are written by the LWS tick's kernels on the engine's stream (ordered before this kernel by an
// event): ld.global.cg, and no L1 allocation for gathers nothing else in the kernel re-reads.
__device__ __forceinline__ int linked_ready(const DsTickArgs& a, uint32_t row, bool exists, int own,
                                            uint32_t& took, uint32_t& fell) {
  const uint4 l = ldg_stream(a.links + row);  // {uid lo, uid hi, lws_row, reserved}
  if (l.z == LWSE_NONE) return own;
  if (exists && l.z < a.n_lws) {
    const uint64_t uid = __ldcg(reinterpret_cast<const unsigned long long*>(&a.lws[l.z].uid_hash));
    if (uid == u64_of(l.x, l.y)) {
      const uint32_t f = __ldcg(&a.lws_out[l.z].flags);
      constexpr uint32_t kNoUpdate = LWSE_LOUT_IRREGULAR | LWSE_LOUT_BAD_TABLE | LWSE_LOUT_RUP_ERROR | LWSE_LOUT_STATUS_ERROR;
      if (!(f & kNoUpdate)) {
        took++;
        return __ldcg(&a.lws_out[l.z].ready_replicas);
      }
    }
  }
  fell++;
  return own;
}

// After the sweep of DS d: list it when its ds_out row, a role_out row or a revrole_out row of its
// ranges differs from the previous tick, when the scatter patched its own row, or on the first tick;
// a listed DS's rows go to the pinned mirrors.  A BAD_TABLE row's ranges are not read.  The
// kernel runs this in a second pass over the same rows (one thread owns the same DS in both), so
// that nothing of it is live across the sweep's registers.
__device__ __forceinline__ void ds_tick_diff(const lwse_ds_tables& t, const DsTickArgs& a, uint32_t d) {
  const uint4 h0 = __ldg(reinterpret_cast<const uint4*>(t.ds + d) + 0);
  const uint4 h1 = __ldg(reinterpret_cast<const uint4*>(t.ds + d) + 1);
  const uint32_t role_base = h0.z, n = h0.w, rev_base = h1.y, nrr = (h1.z + 1u) * h0.w;
  const uint8_t mark = a.marks[d];
  if (mark) a.marks[d] = 0;
  bool changed = a.all || mark;
  const uint4 cur = *reinterpret_cast<const uint4*>(t.ds_out + d);
  const bool bad = cur.x & LWSE_DOUT_BAD_TABLE;
  if (!changed) {
    const uint4 prev = __ldg(reinterpret_cast<const uint4*>(a.prev_ds_out + d));
    changed = cur.x != prev.x || cur.y != prev.y || cur.z != prev.z || cur.w != prev.w;
  }
  const uint2* ro = reinterpret_cast<const uint2*>(t.role_out + role_base);
  const uint2* pro = reinterpret_cast<const uint2*>(a.prev_role_out + role_base);
  const int* rro = t.revrole_out + rev_base;
  const int* prro = a.prev_revrole_out + rev_base;
  if (!bad) {
    for (uint32_t i = 0; i < n && !changed; i++) {
      const uint2 x = ro[i], y = __ldg(pro + i);
      changed = x.x != y.x || x.y != y.y;
    }
    for (uint32_t i = 0; i < nrr && !changed; i++) changed = rro[i] != __ldg(prro + i);
  }
  if (!changed) return;
  *reinterpret_cast<uint4*>(a.m_ds_out + d) = cur;
  if (!bad) {
    uint2* mro = reinterpret_cast<uint2*>(a.m_role_out + role_base);
    for (uint32_t i = 0; i < n; i++) mro[i] = ro[i];
    int* mrro = a.m_revrole_out + rev_base;
    for (uint32_t i = 0; i < nrr; i++) mrro[i] = rro[i];
  }
  // warp-aggregated append: one atomic per warp and call site
  const unsigned m = __activemask();
  const unsigned lane = threadIdx.x & 31u;
  const int leader = __ffs(m) - 1;
  uint32_t base = 0;
  if ((int)lane == leader) base = atomicAdd(a.count, (uint32_t)__popc(m));
  base = __shfl_sync(m, base, leader);
  a.rows[base + __popc(m & ((1u << lane) - 1u))] = d;
}

// How the sweep body reads revision-role rows.  The sweep and the tick read input tables that
// nothing in the kernel writes: ld.global.nc.  The forecast rewrites its scratch copy of the rows
// between the cycles of one kernel, so it reads them with coherent loads, ordered after the thread's
// own stores (the memory clobber: the compiler moves no store of a row past them).
struct RrLoadNc {
  static __device__ __forceinline__ uint4 row(const uint4* p) { return ldg_stream(p); }
  static __device__ __forceinline__ uint32_t flags(const uint32_t* p) { return __ldg(p); }
};
struct RrLoadCoherent {
  static __device__ __forceinline__ uint4 row(const uint4* p) {
    uint4 r;
    asm volatile("ld.global.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p)
                 : "memory");
    return r;
  }
  static __device__ __forceinline__ uint32_t flags(const uint32_t* p) {
    uint32_t r;
    asm volatile("ld.global.u32 %0, [%1];" : "=r"(r) : "l"(p) : "memory");
    return r;
  }
};

// One DS of the sweep (h0, h1: its lwse_ds_rec): writes its ds_out, role_out and revrole_out rows
// and returns {ds_out.flags, ds_out.drained_revs}.  Shared by the sweep, the tick and the forecast.
template <class Ld, bool kLinked>
__device__ __forceinline__ uint2 ds_sweep_one(const lwse_ds_tables& t, const DsTickArgs& a, const uint32_t d,
                                              const uint4 h0, const uint4 h1, uint32_t& took, uint32_t& fell) {
  const uint32_t role_base = h0.z, n_roles = h0.w, n_spec = h1.x, rev_base = h1.y, n_old = h1.z, dflags = h1.w;
  uint32_t oflags = 0, drained = 0, ready_revs = 0;
  const int n = (int)n_roles, S = (int)n_spec, V = (int)n_old;
  if (!ds_rows_ok(t, h0, h1)) {
    stg_stream(t.ds_out + d, make_uint4(LWSE_DOUT_BAD_TABLE, 0, 0, 0));
    return make_uint2(LWSE_DOUT_BAD_TABLE, 0);
  }
  const lwse_ds_role_rec* roles = t.roles + role_base;
  const uint4* rr = reinterpret_cast<const uint4*>(t.revroles + rev_base);  // {replicas, initial, ready, flags}
  lwse_ds_role_out* ro = t.role_out + role_base;
  lwse_ds_revrole_out* rro = t.revrole_out + rev_base;

  int initial_old[MAXR], cur_old[MAXR], cur_new[MAXR], target[MAXR];
  RuConfig cfg[MAXR];
  for (int i = 0; i < n; i++) initial_old[i] = cur_old[i] = cur_new[i] = target[i] = 0;

  // one pass over the old revisions: totals, cleanup predicate, service readiness, defaults
  int total_old_spec = 0;
  for (int r = 0; r < V; r++) {
    bool any = false, all_drained = true, ready = true;
    for (int i = 0; i < n; i++) {
      uint4 x = Ld::row(rr + r * n + i);
      const bool exists = x.w & LWSE_RR_EXISTS;
      if constexpr (kLinked) x.z = (uint32_t)linked_ready(a, rev_base + r * n + i, exists, (int)x.z, took, fell);
      rro[r * n + i] = exists ? (int)x.x : -1;
      if (i < S && (!exists || (int)x.z < 1)) ready = false;  // service_manager.go:62-67
      if (!exists) continue;
      any = true;
      if (((x.w & LWSE_RR_REPLICAS_NIL) ? 0 : (int)x.x) != 0) all_drained = false;  // :222-225
      cur_old[i] += (int)x.x;                                                        // utils.go:167-175
      initial_old[i] += (int)x.y >= 0 ? (int)x.y : (int)x.x;                         // utils.go:177-190
      if (i < S) total_old_spec += (int)x.x;
    }
    if (any && all_drained) drained |= 1u << r;
    if (ready) ready_revs |= 1u << r;
  }
  bool new_ready = true, stable = true;
  for (int i = 0; i < n; i++) {
    uint4 x = Ld::row(rr + V * n + i);
    const bool exists = x.w & LWSE_RR_EXISTS;
    if constexpr (kLinked) x.z = (uint32_t)linked_ready(a, rev_base + V * n + i, exists, (int)x.z, took, fell);
    rro[V * n + i] = exists ? (int)x.x : -1;
    const uint4 rl = ldg_cached(reinterpret_cast<const uint4*>(roles + i));  // {target, surge, unavail, flags}
    const bool in_spec = rl.w & LWSE_ROLE_IN_SPEC;
    if (i < S) {
      if (!exists || (int)x.z < 1) new_ready = false;
      if (!exists || (int)x.x != (int)x.z) stable = false;  // isRevisionStable executor.go:270-281
    }
    if (in_spec) {
      if (exists) cur_new[i] = (int)x.x;
      target[i] = (int)rl.x;
    }
    // extractRollingUpdateConfig executor.go:235-260
    cfg[i].ms = 1;
    cfg[i].mu = 0;
    if (in_spec && (rl.w & LWSE_ROLE_HAS_ROLLING_CONFIG)) {
      const int replicas = (int)rl.x;
      const int surge = (rl.w & LWSE_ROLE_SURGE_INVALID)
                            ? 0
                            : scaled_value((int)rl.y, rl.w & LWSE_ROLE_SURGE_IS_PERCENT, replicas, true);
      const int unav = (rl.w & LWSE_ROLE_UNAVAIL_INVALID)
                           ? 0
                           : scaled_value((int)rl.z, rl.w & LWSE_ROLE_UNAVAIL_IS_PERCENT, replicas, false);
      if (unav > 0) {
        cfg[i].mu = unav;
        cfg[i].ms = surge;
      } else if (surge > 0) {
        cfg[i].ms = surge;
      }
    }
    ro[i].next_old = -1;
    ro[i].next_new = -1;
  }
  if (new_ready) oflags |= LWSE_DOUT_NEW_READY;

  if (!(V > 0 && total_old_spec > 0)) {
    // reconcileSimple disaggregatedset_controller.go:137-186
    for (int i = 0; i < S; i++) rro[V * n + i] = target[i];
  } else {
    oflags |= LWSE_DOUT_ROLLING;
    if (!(dflags & LWSE_DS_HAS_NEW_REVISION)) {
      oflags |= LWSE_DOUT_INIT;  // initRollingUpdate executor.go:85-124
      for (int i = 0; i < S; i++) rro[V * n + i] = 0;
    } else if (stable) {
      oflags |= LWSE_DOUT_STABLE;
      int past[MAXR], new_[MAXR];
      if (!compute_next_step(n, initial_old, cur_old, cur_new, target, cfg, past, new_)) {
        oflags |= LWSE_DOUT_COMPLETE;
      } else {
        oflags |= LWSE_DOUT_STEP;
        for (int i = 0; i < n; i++) {
          ro[i].next_old = past[i];
          ro[i].next_new = new_[i];
          // scaleUpNew executor.go:306-328
          if ((__ldg(&roles[i].flags) & LWSE_ROLE_IN_SPEC) && cur_new[i] < new_[i]) rro[V * n + i] = new_[i];
        }
        // scaleDownOld executor.go:330-398, revisions newest-first (:283-302)
        int budget[MAXR];
        for (int i = 0; i < n; i++) budget[i] = cur_old[i] - past[i];
        uint32_t done_mask = 0;
        for (int k = 0; k < V; k++) {
          bool all_zero = true;
          for (int i = 0; i < n; i++)
            if (budget[i] > 0) all_zero = false;
          if (all_zero) break;
          // next newest revision not yet handled (stable: lowest row on equal stamps)
          int r = -1;
          uint32_t best_ts = 0;
          for (int c = 0; c < V; c++) {
            if (done_mask & (1u << c)) continue;
            uint32_t ts = 0;
            for (int i = 0; i < n; i++) {
              const uint32_t w = Ld::flags(&t.revroles[rev_base + c * n + i].flags);
              if (w & LWSE_RR_EXISTS) ts = max(ts, w >> LWSE_RR_TS_SHIFT);
            }
            if (r < 0 || ts > best_ts) {
              r = c;
              best_ts = ts;
            }
          }
          done_mask |= 1u << r;
          int new_rep[MAXR], planned[MAXR];
          uint32_t trig = 0;
          for (int i = 0; i < n; i++) {
            planned[i] = 0;
            new_rep[i] = 0;
            const int rep = rro[r * n + i];
            if (rep < 0) continue;
            const int drain = min(budget[i], rep);
            planned[i] = drain;
            new_rep[i] = rep - drain;
            if (new_rep[i] == 0) trig |= 1u << i;
          }
          for (int i = 0; i < n; i++) {
            const int rep = rro[r * n + i];
            if (rep < 0) continue;
            const int nr = trig ? 0 : new_rep[i];  // coordinated drain :366-373
            if (rep <= nr) continue;
            rro[r * n + i] = nr;
            if ((trig & (1u << i)) || !trig) budget[i] -= planned[i];  // :392-394
          }
        }
      }
    }
  }
  stg_stream(t.ds_out + d, make_uint4(oflags, drained, ready_revs, 0));
  return make_uint2(oflags, drained);
}

// kTick = false: the stateless sweep (lwse_sweep_ds_*), `a` unused.  kTick = true: the resident tick — diff, mirrors, change list, and the publish of
// the count and sequence word by the last CTA (one system-scope release, as publish_lists_kernel).
// kLinked (with kTick): every revision-role row's ready count goes through linked_ready, and the two
// row counts are published beside the changed-row count.
template <bool kTick, bool kLinked = false>
__global__ void __launch_bounds__(128) ds_sweep_kernel(const lwse_ds_tables t, const DsTickArgs a) {
  uint32_t took = 0, fell = 0;
  for (uint32_t d = blockIdx.x * blockDim.x + threadIdx.x; d < t.n_ds; d += gridDim.x * blockDim.x) {
    const uint4 h0 = ldg_stream(reinterpret_cast<const uint4*>(t.ds + d) + 0);
    const uint4 h1 = ldg_stream(reinterpret_cast<const uint4*>(t.ds + d) + 1);
    ds_sweep_one<RrLoadNc, kLinked>(t, a, d, h0, h1, took, fell);
  }
  if constexpr (kTick) {
    for (uint32_t d = blockIdx.x * blockDim.x + threadIdx.x; d < t.n_ds; d += gridDim.x * blockDim.x) ds_tick_diff(t, a, d);
    if constexpr (kLinked) {  // (every lane of the block is here: the loops above have ended)
      took = __reduce_add_sync(0xFFFFFFFFu, took);
      fell = __reduce_add_sync(0xFFFFFFFFu, fell);
      if ((threadIdx.x & 31u) == 0 && (took | fell)) {
        atomicAdd(a.count + 2, took);
        atomicAdd(a.count + 3, fell);
      }
    }
    // the ticket orders every CTA's stores (bar.sync, then a gpu-scope release) before the last
    // CTA's acquire; its system-scope release of the sequence word covers them all
    __shared__ uint32_t s_last;
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t tk;
      asm volatile("atom.add.acq_rel.gpu.global.u32 %0, [%1], 1;" : "=r"(tk) : "l"(a.ticket) : "memory");
      s_last = tk == gridDim.x - 1u ? 1u : 0u;
      if (s_last) {
        volatile uint32_t* hw = a.host_words;
        hw[0] = __ldcg(a.count);
        *a.count = 0u;
        *a.ticket = 0u;
        if constexpr (kLinked) {  // [2] rows that took the LWS value, [3] linked rows that fell back
          hw[2] = __ldcg(a.count + 2);
          hw[3] = __ldcg(a.count + 3);
          a.count[2] = 0u;
          a.count[3] = 0u;
        }
        asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(a.host_words + 1), "r"(a.seq) : "memory");
      }
    }
  }
}

// ---- rollout forecast (lwse_ds_forecast_*): the cycle rules are in lwse.h ----
struct DsForecastArgs {
  lwse_ds_revrole_rec* rows;            // scratch copy of the revision-role table (same row numbers)
  lwse_ds_out* s_ds_out;                // the sweep body's outputs for the replay (scratch)
  lwse_ds_role_out* s_role_out;
  lwse_ds_revrole_out* s_revrole_out;
  lwse_ds_forecast* fc;                 // [n_ds]
  lwse_ds_forecast_role* fc_role;       // [n_roles]
  lwse_ds_role_out* steps;              // [step_capacity] (write pass only)
  uint32_t step_capacity;
  unsigned long long* totals;           // scan: [0] rows needed, [1] rows written
};

__device__ __forceinline__ int clamp32(long long v) {
  return (int)max(min(v, (long long)INT32_MAX), (long long)INT32_MIN);
}

// Per-role old (existing old-revision rows) and new (the new revision's row) counts of a DS's rows.
__device__ __forceinline__ void ds_role_counts(const uint4* rows, int n, int V, long long* old_c, long long* new_c) {
  for (int i = 0; i < n; i++) old_c[i] = new_c[i] = 0;
  for (int r = 0; r <= V; r++)
    for (int i = 0; i < n; i++) {
      const uint4 x = rows[r * n + i];
      if (!(x.w & LWSE_RR_EXISTS)) continue;
      if (r < V)
        old_c[i] += (int)x.x;
      else
        new_c[i] = (int)x.x;
    }
}

// The replay of DS d.  kWrite = false: summaries, and the DS's trajectory row count in step_base
// (the scan turns it into an offset).  kWrite = true: replays the DS again and writes its rows.
// The thread owns the DS's scratch rows, so nothing is shared between threads.
template <bool kWrite>
__device__ void ds_forecast_one(const lwse_ds_tables& in, const DsForecastArgs& f, const uint32_t d) {
  const uint4 h0 = ldg_stream(reinterpret_cast<const uint4*>(in.ds + d) + 0);
  uint4 h1 = ldg_stream(reinterpret_cast<const uint4*>(in.ds + d) + 1);
  if (!ds_rows_ok(in, h0, h1)) {
    if (!kWrite) f.fc[d] = lwse_ds_forecast{LWSE_DSF_BAD_TABLE, 0u, 0u, 0u};
    return;
  }
  // The write pass writes at most the n_steps rows the summary pass counted and the scan reserved
  // below step_capacity.  Its replay finds the same steps, except where DS row ranges overlap (their
  // threads then share scratch rows and the results are unspecified): the bound keeps every store
  // inside the DS's own reserved rows even then.
  uint32_t step_base = 0, step_limit = 0;
  if constexpr (kWrite) {
    const lwse_ds_forecast c = f.fc[d];
    if (c.n_steps == 0 || (c.flags & LWSE_DSF_TRUNCATED)) return;
    step_base = c.step_base;
    step_limit = c.n_steps;
  }
  const uint32_t role_base = h0.z, rev_base = h1.y;
  const int n = (int)h0.w, S = (int)h1.x, V = (int)h1.z, nrr = (V + 1) * n;
  const lwse_ds_role_rec* roles = in.roles + role_base;
  const uint4* src = reinterpret_cast<const uint4*>(in.revroles + rev_base);
  uint4* rows = reinterpret_cast<uint4*>(f.rows + rev_base);  // {replicas, initial, ready, flags}

  // private copy of the rows; the cap's M; the newest creation rank
  long long mx[MAXR];
  for (int i = 0; i < n; i++) mx[i] = 0;
  uint32_t rank = 0;
  for (int k = 0; k < nrr; k++) {
    const uint4 x = ldg_stream(src + k);
    rows[k] = x;
    if (x.w & LWSE_RR_EXISTS) {
      mx[k % n] += max((int)x.x, (int)x.y);
      rank = max(rank, x.w >> LWSE_RR_TS_SHIFT);
    }
  }
  long long M = 0;
  for (int i = 0; i < n; i++) M = max(M, max(mx[i], (long long)__ldg(&roles[i].target_replicas)));
  const uint32_t cap = (uint32_t)min(2 * M + 12, (long long)LWSE_DS_FORECAST_MAX_CYCLES);

  long long old_c[MAXR], new_c[MAXR], peak[MAXR], floor_[MAXR];
  ds_role_counts(rows, n, V, old_c, new_c);
  for (int i = 0; i < n; i++) peak[i] = floor_[i] = old_c[i] + new_c[i];

  lwse_ds_tables t = in;
  t.revroles = f.rows;
  t.ds_out = f.s_ds_out;
  t.role_out = f.s_role_out;
  t.revrole_out = f.s_revrole_out;
  const DsTickArgs none{};
  uint32_t unused = 0;
  // the current rows as they are: the rolling path, and whether the new revision is stable
  const uint2 now = ds_sweep_one<RrLoadCoherent, false>(t, none, d, h0, h1, unused, unused);
  uint32_t flags = 0, cycles = 0, n_steps = 0;
  const lwse_ds_revrole_out* rro = f.s_revrole_out + rev_base;
  if (now.x & LWSE_DOUT_ROLLING) {
    flags = LWSE_DSF_ROLLING;
    if (!(now.x & (LWSE_DOUT_INIT | LWSE_DOUT_STABLE))) flags |= LWSE_DSF_WAITING;
    bool stopped = false;
    for (uint32_t c = 0; c < cap; c++) {
      for (int k = 0; k < nrr; k++) {  // 1. every child ready
        uint4 x = rows[k];
        if (x.w & LWSE_RR_EXISTS) {
          x.z = x.x;
          rows[k] = x;
        }
      }
      const uint2 o = ds_sweep_one<RrLoadCoherent, false>(t, none, d, h0, h1, unused, unused);  // 2.
      bool changed = false;
      for (int r = 0; r < V; r++) {  // 3. cleanupDrainedLWS
        if (!((o.y >> r) & 1u)) continue;
        changed = true;
        for (int i = 0; i < n; i++) {
          uint4 x = rows[r * n + i];
          x.w &= ~LWSE_RR_EXISTS;
          rows[r * n + i] = x;
        }
      }
      if (o.x & LWSE_DOUT_INIT) {  // 4. initRollingUpdate
        changed = true;
        h1.w |= LWSE_DS_HAS_NEW_REVISION;
        for (int k = 0; k < V * n; k++) {
          uint4 x = rows[k];
          if (x.w & LWSE_RR_EXISTS) {
            x.y = x.x;
            rows[k] = x;
          }
        }
      }
      for (int k = 0; k < nrr; k++) {  // 5. the decided replicas
        const int v = rro[k];
        if (v < 0) continue;
        uint4 x = rows[k];
        if (x.w & LWSE_RR_EXISTS) {
          if ((int)x.x == v && !(x.w & LWSE_RR_REPLICAS_NIL)) continue;
          x.x = (uint32_t)v;
          x.w &= ~LWSE_RR_REPLICAS_NIL;
        } else if (k >= V * n) {
          x = make_uint4((uint32_t)v, 0xFFFFFFFFu, 0u, LWSE_RR_EXISTS | (rank << LWSE_RR_TS_SHIFT));
        } else {
          continue;
        }
        rows[k] = x;
        changed = true;
      }
      if (!changed) {
        stopped = true;
        break;
      }
      cycles++;
      long long nold[MAXR], nnew[MAXR];
      ds_role_counts(rows, n, V, nold, nnew);
      bool step = false;
      for (int i = 0; i < n; i++) {
        if (nold[i] != old_c[i] || nnew[i] != new_c[i]) step = true;
        peak[i] = max(peak[i], old_c[i] + nnew[i]);
        floor_[i] = min(floor_[i], nold[i] + new_c[i]);
        old_c[i] = nold[i];
        new_c[i] = nnew[i];
      }
      if (step) {
        if constexpr (kWrite) {
          uint2* out = reinterpret_cast<uint2*>(f.steps + step_base + n_steps * (uint32_t)n);
          for (int i = 0; i < n; i++) out[i] = make_uint2((uint32_t)clamp32(nold[i]), (uint32_t)clamp32(nnew[i]));
        }
        n_steps++;
        if constexpr (kWrite) {
          if (n_steps == step_limit) return;  // every reserved row is written: the rest is the summary pass's
        }
      }
    }
    bool done = stopped;
    for (int i = 0; i < n; i++) {
      if (old_c[i] != 0) done = false;
      if (i < S && new_c[i] != (long long)__ldg(&roles[i].target_replicas)) done = false;
    }
    flags |= done ? LWSE_DSF_DONE : LWSE_DSF_UNFINISHED;
  }
  if constexpr (!kWrite) {
    f.fc[d] = lwse_ds_forecast{flags, cycles, n_steps * (uint32_t)n, n_steps};
    for (int i = 0; i < n; i++)
      f.fc_role[role_base + i] =
          lwse_ds_forecast_role{clamp32(peak[i]), clamp32(floor_[i]), clamp32(old_c[i]), clamp32(new_c[i])};
  }
}

template <bool kWrite>
__global__ void __launch_bounds__(128) ds_forecast_kernel(const lwse_ds_tables in, const DsForecastArgs f) {
  for (uint32_t d = blockIdx.x * blockDim.x + threadIdx.x; d < in.n_ds; d += gridDim.x * blockDim.x)
    ds_forecast_one<kWrite>(in, f, d);
}

// write_pass = false: the summary pass and the scan.  write_pass = true: the write pass into h->steps,
// which holds the rows the scan counted as written.  Both on stream s.
int launch_ds_forecast(const lwse_ds_tables* t, const DsForecastHost* h, bool write_pass, int sm_count, cudaStream_t s) {
  if (t->n_ds == 0) return 0;
  const uint32_t want = (t->n_ds + 127u) / 128u;
  const uint32_t cap = (uint32_t)sm_count * 16u;
  const uint32_t grid = want < cap ? want : cap;
  const DsForecastArgs f{h->rows, h->s_ds_out, h->s_role_out, h->s_revrole_out, h->fc, h->fc_role,
                         h->steps, h->step_capacity, h->totals};
  int launched;
  if (write_pass) {
    ds_forecast_kernel<true><<<grid, 128, 0, s>>>(*t, f);
    launched = 1;
  } else {
    ds_forecast_kernel<false><<<grid, 128, 0, s>>>(*t, f);
    // (totals[2..] holds the scan's block sums)
    launch_forecast_scan(StepLayoutOp<lwse_ds_forecast, LWSE_DSF_TRUNCATED>{h->fc, h->step_capacity, h->want_steps ? 1 : 0},
                         t->n_ds, h->totals + 2, h->totals + 0, h->totals + 1, s);
    launched = 4;
  }
  return launch_result(launched);
}

int launch_ds_sweep(const lwse_ds_tables* t, int sm_count, cudaStream_t s) {
  if (t->n_ds == 0) return 0;
  const uint32_t want = (t->n_ds + 127u) / 128u;
  const uint32_t cap = (uint32_t)sm_count * 16u;
  ds_sweep_kernel<false><<<want < cap ? want : cap, 128, 0, s>>>(*t, DsTickArgs{});
  return launch_result(1);
}

int launch_ds_tick(const lwse_ds_tables* t, const DsTickHost* h, int sm_count, cudaStream_t s) {
  if (t->n_ds == 0) return 0;
  const uint32_t want = (t->n_ds + 127u) / 128u;
  const uint32_t cap = (uint32_t)sm_count * 16u;
  const DsTickArgs a{h->prev_ds_out, h->prev_role_out, h->prev_revrole_out, h->m_ds_out, h->m_role_out, h->m_revrole_out,
                     h->marks, h->rows, h->counters, h->counters + 1, h->host_words, h->seq, h->all ? 1u : 0u,
                     h->links, h->lws, h->lws_out, h->n_lws};
  if (h->links)
    ds_sweep_kernel<true, true><<<want < cap ? want : cap, 128, 0, s>>>(*t, a);
  else
    ds_sweep_kernel<true><<<want < cap ? want : cap, 128, 0, s>>>(*t, a);
  return launch_result(1);
}

// ---- DS drain (lwse_resident_ds_drain*): the definitions are in lwse.h ----
//   ds_sweep_kernel<false, true>  the before and the after sweep: the linked sweep body without the tick's
//                                 diff, mirrors and publish, reading ready counts from the baseline lws_out or
//                                 from its copy with the drain's lost groups taken off.
//   ds_drain_diff_kernel          one thread per DS: its rows' link rule against lost[L] (rows touched / zeroed
//                                 / linked), the two sweeps' rows compared, the verdicts; touched DS appended
//                                 with one atomic per warp, the totals reduced per warp.
//   ds_drain_links_kernel         the per-key form's reverse link index (count, then fill behind the scan).
static unsigned ds_grid(uint32_t n_ds, int sm_count) {
  const uint32_t want = (n_ds + 127u) / 128u, cap = (uint32_t)sm_count * 16u;
  return want < cap ? want : cap;
}

// The LWS row whose ready count revision-role row `row` takes under the link rule (linked_ready), or LWSE_NONE.
__device__ __forceinline__ uint32_t ds_drain_link_of(const DsDrainLink& lk, uint32_t row, bool exists) {
  return ds_link_target(lk.links, lk.lws, lk.lws_out, lk.n_lws, row, exists);
}

__device__ __forceinline__ bool u4_ne(const uint4 a, const uint4 b) { return a.x != b.x || a.y != b.y || a.z != b.z || a.w != b.w; }

__global__ void __launch_bounds__(128, 4) ds_drain_diff_kernel(const lwse_ds_tables t, const DsDrainLink lk, const DsDrainDiffHost h) {
  uint32_t service = 0, old_service = 0, stalled = 0, changed_n = 0, rows_touched = 0, rows_zeroed = 0, linked = 0;
  const uint32_t lane = threadIdx.x & 31u;
  for (uint32_t d = blockIdx.x * blockDim.x + threadIdx.x; d < t.n_ds; d += gridDim.x * blockDim.x) {
    const uint4 h0 = ldg_stream(reinterpret_cast<const uint4*>(t.ds + d) + 0);
    const uint4 h1 = ldg_stream(reinterpret_cast<const uint4*>(t.ds + d) + 1);
    const uint4 after = __ldcg(reinterpret_cast<const uint4*>(t.ds_out + d));
    const uint4 before = __ldcg(reinterpret_cast<const uint4*>(h.before_ds_out + d));
    bool changed = u4_ne(after, before);
    uint32_t touched = 0, zeroed = 0, new_zeroed = 0, old_zeroed = 0;
    if (!(before.x & LWSE_DOUT_BAD_TABLE)) {  // (BAD_TABLE in both sweeps, or in neither)
      const uint32_t role_base = h0.z, n = h0.w, S = h1.x, rev_base = h1.y, V = h1.z, nrr = (h1.z + 1u) * h0.w;
      const uint32_t fell = before.z & ~after.z;  // old revisions whose service the drain takes down
      for (uint32_t k = 0; k < nrr; k++) {
        const uint32_t row = rev_base + k;
        const uint32_t L = ds_drain_link_of(lk, row, __ldg(&t.revroles[row].flags) & LWSE_RR_EXISTS);
        if (L == LWSE_NONE) continue;
        linked++;
        const uint32_t lost = __ldg(h.lost + L);
        if (lost == 0) continue;
        touched++;
        const int32_t rb = __ldg(&lk.lws_out[L].ready_replicas);
        const int64_t ra = (int64_t)rb - lost;
        if (!(rb >= 1 && ra < 1)) continue;
        zeroed++;
        const uint32_t r = k / n, i = k - r * n;
        if (i >= S) continue;  // (a removed role serves nothing)
        if (r == V)
          new_zeroed |= 1u << i;
        else if ((fell >> r) & 1u)
          old_zeroed |= 1u << i;
      }
      const uint2* ro = reinterpret_cast<const uint2*>(t.role_out + role_base);
      const uint2* pro = reinterpret_cast<const uint2*>(h.before_role_out + role_base);
      for (uint32_t i = 0; i < n && !changed; i++) {
        const uint2 x = __ldcg(ro + i), y = __ldcg(pro + i);
        changed = x.x != y.x || x.y != y.y;
      }
      for (uint32_t i = 0; i < nrr && !changed; i++)
        changed = __ldcg(t.revrole_out + rev_base + i) != __ldcg(h.before_revrole_out + rev_base + i);
    }
    if (touched == 0) continue;  // (only the ready column of touched rows differs: an untouched DS is unchanged)
    uint32_t flags = LWSE_DSD_TOUCHED;
    if ((before.x & LWSE_DOUT_NEW_READY) && !(after.x & LWSE_DOUT_NEW_READY)) flags |= LWSE_DSD_SERVICE_LOST;
    if (before.z & ~after.z) flags |= LWSE_DSD_OLD_SERVICE_LOST;
    if ((before.x & LWSE_DOUT_STABLE) && !(after.x & LWSE_DOUT_STABLE)) flags |= LWSE_DSD_STALLS;
    if (changed) flags |= LWSE_DSD_CHANGED;
    service += (flags & LWSE_DSD_SERVICE_LOST) ? 1u : 0u;
    old_service += (flags & LWSE_DSD_OLD_SERVICE_LOST) ? 1u : 0u;
    stalled += (flags & LWSE_DSD_STALLS) ? 1u : 0u;
    changed_n += changed ? 1u : 0u;
    rows_touched += touched;
    rows_zeroed += zeroed;
    // warp-aggregated append: one atomic per warp
    const unsigned m = __activemask();
    const int leader = __ffs(m) - 1;
    uint32_t at = 0;
    if ((int)lane == leader) at = atomicAdd(h.counts + 16, (uint32_t)__popc(m));
    at = __shfl_sync(m, at, leader) + (uint32_t)__popc(m & ((1u << lane) - 1u));
    if (at < h.capacity) {
      uint4* out = reinterpret_cast<uint4*>(h.rows + at);
      out[0] = make_uint4(d, flags, touched, zeroed);
      out[1] = make_uint4(new_zeroed, old_zeroed, 0u, 0u);
      out[2] = before;
      out[3] = after;
    }
  }
  // (every lane of the warp is here: the loop above has ended)
  service = __reduce_add_sync(0xFFFFFFFFu, service);
  old_service = __reduce_add_sync(0xFFFFFFFFu, old_service);
  stalled = __reduce_add_sync(0xFFFFFFFFu, stalled);
  changed_n = __reduce_add_sync(0xFFFFFFFFu, changed_n);
  rows_touched = __reduce_add_sync(0xFFFFFFFFu, rows_touched);
  rows_zeroed = __reduce_add_sync(0xFFFFFFFFu, rows_zeroed);
  linked = __reduce_add_sync(0xFFFFFFFFu, linked);
  if (lane != 0) return;
  if (service) atomicAdd(h.counts + 17, service);
  if (old_service) atomicAdd(h.counts + 18, old_service);
  if (stalled) atomicAdd(h.counts + 19, stalled);
  if (changed_n) atomicAdd(h.counts + 20, changed_n);
  if (rows_touched) atomicAdd(h.counts + 21, rows_touched);
  if (rows_zeroed) atomicAdd(h.counts + 22, rows_zeroed);
  if (linked) atomicAdd(h.counts + 23, linked);
}

// kFill = false: count[L] += the rows that take L's value, and *total (64-bit) += every such row (the entries the
// fill writes: a row in the ranges of several DS counts once per DS).  kFill = true: each row's entry at
// cursor[L]++, written only below capacity (the caller sized `entries` from *total, so every entry fits).
template <bool kFill>
__global__ void __launch_bounds__(128) ds_drain_links_kernel(const lwse_ds_tables t, const DsDrainLink lk, uint32_t* count,
                                                            uint32_t* cursor, uint4* entries, uint32_t capacity,
                                                            unsigned long long* total) {
  unsigned long long rows = 0;
  for (uint32_t d = blockIdx.x * blockDim.x + threadIdx.x; d < t.n_ds; d += gridDim.x * blockDim.x) {
    const uint4 h0 = ldg_stream(reinterpret_cast<const uint4*>(t.ds + d) + 0);
    const uint4 h1 = ldg_stream(reinterpret_cast<const uint4*>(t.ds + d) + 1);
    if (!ds_rows_ok(t, h0, h1)) continue;
    const uint32_t n = h0.w, S = h1.x, rev_base = h1.y, V = h1.z;
    for (uint32_t r = 0; r <= V; r++)
      for (uint32_t i = 0; i < n; i++) {
        const uint32_t row = rev_base + r * n + i;
        const uint32_t L = ds_drain_link_of(lk, row, __ldg(&t.revroles[row].flags) & LWSE_RR_EXISTS);
        if (L == LWSE_NONE) continue;
        if (!kFill) {
          atomicAdd(count + L, 1u);
          rows++;
        } else {
          const uint32_t at = atomicAdd(cursor + L, 1u);
          const uint32_t info = (r == V ? kDsDrainNewSlot : r) | (i < S ? kDsDrainSpec : 0u);
          if (at < capacity) entries[at] = make_uint4(d, info, (uint32_t)__ldg(&lk.lws_out[L].ready_replicas), 0u);
        }
      }
  }
  if (!kFill) {
    // (every lane of the warp is here: the loop above has ended)
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) rows += __shfl_xor_sync(0xFFFFFFFFu, rows, off);
    if ((threadIdx.x & 31u) == 0 && rows) atomicAdd(total, rows);
  }
}

int launch_ds_drain_sweep(const lwse_ds_tables* t, const DsDrainLink* lk, const lwse_lws_out* ready_from, int sm_count,
                          cudaStream_t s) {
  if (t->n_ds == 0) return 0;
  DsTickArgs a{};
  a.links = lk->links;
  a.lws = lk->lws;
  a.lws_out = ready_from;
  a.n_lws = lk->n_lws;
  ds_sweep_kernel<false, true><<<ds_grid(t->n_ds, sm_count), 128, 0, s>>>(*t, a);
  return launch_result(1);
}

int launch_ds_drain_diff(const lwse_ds_tables* t, const DsDrainLink* lk, const DsDrainDiffHost* h, int sm_count,
                         cudaStream_t s) {
  if (t->n_ds == 0) return 0;
  ds_drain_diff_kernel<<<ds_grid(t->n_ds, sm_count), 128, 0, s>>>(*t, *lk, *h);
  return launch_result(1);
}

int launch_ds_drain_links(const lwse_ds_tables* t, const DsDrainLink* lk, uint32_t* count, uint32_t* cursor, uint4* entries,
                          uint32_t capacity, unsigned long long* total, bool fill, int sm_count, cudaStream_t s) {
  if (t->n_ds == 0) return 0;
  if (fill)
    ds_drain_links_kernel<true><<<ds_grid(t->n_ds, sm_count), 128, 0, s>>>(*t, *lk, count, cursor, entries, capacity, total);
  else
    ds_drain_links_kernel<false><<<ds_grid(t->n_ds, sm_count), 128, 0, s>>>(*t, *lk, count, cursor, entries, capacity, total);
  return launch_result(1);
}

}  // namespace lwse
