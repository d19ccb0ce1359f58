// Shared device helpers for the lwse kernels (sm_90a).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <utility>

#include "../../include/lwse.h"

namespace lwse {

constexpr int kSmCount = 132;  // H100 SXM

// L2 eviction policy for the small tables every tick reads again (node table and its index,
// placement requests, occupancy): evict_last, so that the tens of MB a sweep streams through L2
// go first.  (createpolicy; the asm is not volatile, so identical requests in one kernel fold
// into one instruction.)  It is a guard for sweeps that stream more than the 50 MB of L2, not a
// speed-up on its own.
__device__ __forceinline__ uint64_t policy_evict_last() {
  uint64_t pol;
  asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}

// 128-bit streaming load: read-only path, do not allocate in L1 (each row is consumed once per
// sweep).  (No L2 evict_first hint on top: the group pass re-reads the state words of event pods,
// which would then come from DRAM again.)
__device__ __forceinline__ uint4 ldg_stream(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

// Loads of small tables that every tick reads again: last to go in L2.
__device__ __forceinline__ uint4 ldg_keep(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p), "l"(policy_evict_last()));
  return r;
}
__device__ __forceinline__ uint32_t ldg_keep_u32(const uint32_t* p) {
  uint32_t r;
  asm volatile("ld.global.nc.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(r) : "l"(p), "l"(policy_evict_last()));
  return r;
}

// 128-bit load through L1 (rows shared by neighbouring tiles: owner rows, node rows).
__device__ __forceinline__ uint4 ldg_cached(const void* p) {
  return __ldg(reinterpret_cast<const uint4*>(p));
}

__device__ __forceinline__ void stg_stream(void* p, uint4 v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y),
               "r"(v.z), "r"(v.w)
               : "memory");
}

__device__ __forceinline__ uint64_t u64_of(uint32_t lo, uint32_t hi) {
  return (uint64_t)lo | ((uint64_t)hi << 32);
}

// Lane mask of the W-wide tile this lane belongs to.
template <int W>
__device__ __forceinline__ uint32_t tile_mask() {
  if constexpr (W == 32) {
    return 0xFFFFFFFFu;
  } else {
    const uint32_t lane = threadIdx.x & 31u;
    return ((1u << W) - 1u) << (lane & ~(uint32_t)(W - 1));
  }
}

template <int W>
__device__ __forceinline__ uint32_t tile_or(uint32_t v) {
  if constexpr (W == 1) return v;
  return __reduce_or_sync(tile_mask<W>(), v);
}
template <int W>
__device__ __forceinline__ uint32_t tile_min(uint32_t v) {
  if constexpr (W == 1) return v;
  return __reduce_min_sync(tile_mask<W>(), v);
}
template <int W>
__device__ __forceinline__ int32_t tile_max(int32_t v) {
  if constexpr (W == 1) return v;
  return __reduce_max_sync(tile_mask<W>(), v);
}
template <int W>
__device__ __forceinline__ int32_t tile_add(int32_t v) {
  if constexpr (W == 1) return v;
  return __reduce_add_sync(tile_mask<W>(), v);
}

// intstr.GetScaledValueFromIntOrPercent in integers.  The reference evaluates
// ceil/floor(float64(v)*float64(total)/100); for |v*total| < 2^53 the float
// quotient is on the same side of every integer as the exact one, so integer
// floor/ceil division gives the identical result (DESIGN.md, "float vs int").
__device__ __forceinline__ int32_t scaled_value(int32_t val, bool is_percent, int32_t total,
                                                bool round_up) {
  if (!is_percent) return val;
  const int64_t num = (int64_t)val * (int64_t)total;
  int64_t q = num / 100;
  const int64_t r = num - q * 100;
  if (r != 0) {
    if (round_up && num > 0) q += 1;
    if (!round_up && num < 0) q -= 1;
  }
  return (int32_t)q;
}

// The table checks of one DS (BAD_TABLE when they fail): its ranges lie inside the tables.  The DS sweep,
// tick, forecast and drain, and the DS rollout what-if, which decides the same way for a proposal.
__device__ __forceinline__ bool ds_rows_ok(const lwse_ds_tables& t, const uint4 h0, const uint4 h1) {
  const uint32_t role_base = h0.z, n_roles = h0.w, n_spec = h1.x, rev_base = h1.y, n_old = h1.z;
  return !(n_roles > LWSE_DS_MAX_ROLES || n_spec > n_roles || n_old > LWSE_DS_MAX_OLD_REVS ||
           (uint64_t)role_base + n_roles > t.n_roles ||
           (uint64_t)rev_base + (uint64_t)(n_old + 1u) * n_roles > t.n_revroles);
}

// Programmatic dependent launch (PDL): the kernels of one sweep are launched
// with programmatic stream serialization, call pdl_launch_dependents() first
// thing (the next kernel may start its own prologue) and pdl_wait_prior()
// right before the first access to data the previous kernel produces.
__device__ __forceinline__ void pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
__device__ __forceinline__ void pdl_wait_prior() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---- the trajectory layout of the rollout forecasts (lwse_ds_forecast_*, lwse_lws_forecast_*) ----
constexpr int kForecastScanThreads = 1024;

// Exclusive prefix over one CTA of kForecastScanThreads threads of one value per thread.
__device__ __forceinline__ unsigned long long cta_exclusive_scan(const unsigned long long sum) {
  __shared__ unsigned long long s_warp[kForecastScanThreads / 32];
  const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  unsigned long long incl = sum;
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long v = __shfl_up_sync(0xFFFFFFFFu, incl, o);
    if ((int)lane >= o) incl += v;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    unsigned long long w = s_warp[lane], wi = w;
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long v = __shfl_up_sync(0xFFFFFFFFu, wi, o);
      if ((int)lane >= o) wi += v;
    }
    s_warp[lane] = wi - w;
  }
  __syncthreads();
  return s_warp[warp] + incl - sum;
}

// An exclusive prefix over n items in three launches (Op::count(i) = item i's count):
//   scan_block_sums_kernel  one CTA per kForecastScanThreads consecutive items (coalesced): their sum
//   scan_carry_kernel       one CTA: the block sums become exclusive block offsets; *total = the sum
//   scan_apply_kernel       every item's offset to Op::apply(i, offset, count), whose results are summed
//                           into *acc (nullable; the sum of one warp must fit 32 bits)
// sums: forecast_scan_words(n) words of device scratch.
inline uint32_t forecast_scan_words(uint32_t n) { return (n + kForecastScanThreads - 1) / kForecastScanThreads; }

template <class Op>
__global__ void __launch_bounds__(kForecastScanThreads) scan_block_sums_kernel(const Op op, uint32_t n,
                                                                               unsigned long long* sums) {
  const uint32_t i = blockIdx.x * kForecastScanThreads + threadIdx.x;
  const unsigned long long v = i < n ? op.count(i) : 0ull;
  const unsigned long long ex = cta_exclusive_scan(v);
  if (threadIdx.x == kForecastScanThreads - 1) sums[blockIdx.x] = ex + v;
}

template <class Op>  // (only to give each user its own instance)
__global__ void __launch_bounds__(kForecastScanThreads) scan_carry_kernel(unsigned long long* sums, uint32_t n_blocks,
                                                                          unsigned long long* total) {
  __shared__ unsigned long long s_chunk;
  unsigned long long carry = 0;
  for (uint32_t b0 = 0; b0 < n_blocks; b0 += kForecastScanThreads) {
    const uint32_t b = b0 + threadIdx.x;
    const unsigned long long v = b < n_blocks ? sums[b] : 0ull;
    const unsigned long long ex = cta_exclusive_scan(v);
    if (b < n_blocks) sums[b] = carry + ex;
    if (threadIdx.x == kForecastScanThreads - 1) s_chunk = ex + v;
    __syncthreads();
    carry += s_chunk;
    __syncthreads();  // (s_chunk and the scan's shared words are rewritten by the next chunk)
  }
  if (threadIdx.x == 0) *total = carry;
}

template <class Op>
__global__ void __launch_bounds__(kForecastScanThreads) scan_apply_kernel(const Op op, uint32_t n,
                                                                          const unsigned long long* sums,
                                                                          unsigned long long* acc) {
  const uint32_t i = blockIdx.x * kForecastScanThreads + threadIdx.x;
  const unsigned long long v = i < n ? op.count(i) : 0ull;
  const unsigned long long base = cta_exclusive_scan(v) + sums[blockIdx.x];
  const unsigned long long r = i < n ? op.apply(i, base, v) : 0ull;
  if (acc != nullptr) {
    const unsigned w = __reduce_add_sync(0xFFFFFFFFu, (unsigned)r);
    if ((threadIdx.x & 31u) == 0 && w) atomicAdd(acc, (unsigned long long)w);
  }
}

// Enqueues the scan's kernels (three, one when n is 0); the caller checks them with the launches around.
template <class Op>
inline void launch_forecast_scan(const Op& op, uint32_t n, unsigned long long* sums, unsigned long long* total,
                                 unsigned long long* acc, cudaStream_t s) {
  const uint32_t blocks = forecast_scan_words(n);
  if (blocks) scan_block_sums_kernel<Op><<<blocks, kForecastScanThreads, 0, s>>>(op, n, sums);
  scan_carry_kernel<Op><<<1, kForecastScanThreads, 0, s>>>(sums, blocks, total);
  if (blocks) scan_apply_kernel<Op><<<blocks, kForecastScanThreads, 0, s>>>(op, n, sums, acc);
}

// The trajectory layout: step_base (a row count after the summary pass) becomes the exclusive prefix over
// the objects in row order, saturated to 32 bits; with a trajectory buffer, objects whose rows end beyond
// step_capacity get kTruncated.  Total: rows needed; acc: rows written (< 2^32: bounded by capacity).
template <class Rec, uint32_t kTruncated>
struct StepLayoutOp {
  Rec* fc;
  uint32_t capacity;
  int has_steps;
  __device__ __forceinline__ unsigned long long count(uint32_t i) const { return fc[i].step_base; }
  __device__ __forceinline__ unsigned long long apply(uint32_t i, unsigned long long base,
                                                      unsigned long long rows) const {
    Rec c = fc[i];
    c.step_base = (uint32_t)min(base, 0xFFFFFFFFull);
    unsigned long long written = 0;
    if (has_steps && rows) {
      if (base + rows > capacity)
        c.flags |= kTruncated;
      else
        written = rows;
    }
    fc[i] = c;
    return written;
  }
};

// A grid of one CTA per per_cta items, at least one CTA and at most cap.
inline unsigned grid_for(uint64_t items, uint32_t per_cta, uint32_t cap) {
  uint64_t grid = (items + per_cta - 1) / per_cta;
  if (grid < 1) grid = 1;
  return (unsigned)(grid < cap ? grid : cap);
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s,
                              bool pdl, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

// The drain placement (lwse_resident_drain_place_cost): one row's contribution, baseline o and what-if v, to
// words 2..10 of its key's lwse_drain_place_cost row (the three totals as deltas).
constexpr uint32_t kDrainCounts = 9;  // stranded, bumped, changed, lost, moved, gained, PLACED, UNSCHED., CONFLICT
__device__ __forceinline__ void drain_place_count(uint32_t* c, const uint4 o, const uint4 v, bool unpinned) {
  const bool was = (o.z & LWSE_PLACE_PLACED) != 0u, is = (v.z & LWSE_PLACE_PLACED) != 0u;
  c[0] += (unpinned && !is) ? 1u : 0u;
  c[1] += (!unpinned && was && !is) ? 1u : 0u;
  c[2] += (v.x != o.x || v.y != o.y || v.z != o.z || v.w != o.w) ? 1u : 0u;
  c[3] += (was && !is) ? 1u : 0u;
  c[4] += (was && is && o.x != v.x) ? 1u : 0u;
  c[5] += (!was && is) ? 1u : 0u;
  c[6] += (uint32_t)is - (uint32_t)was;
  c[7] += ((v.z & LWSE_PLACE_UNSCHEDULABLE) ? 1u : 0u) - ((o.z & LWSE_PLACE_UNSCHEDULABLE) ? 1u : 0u);
  c[8] += ((v.z & LWSE_PLACE_CONFLICT) ? 1u : 0u) - ((o.z & LWSE_PLACE_CONFLICT) ? 1u : 0u);
}

// What the budget of one LWS row needs from its row and its baseline result row.
// (lwse_drain_kernels.cu and lwse_drain_wave_kernels.cu: the drain budget's definition in lwse.h.)
struct LwsBudget {
  uint32_t gbase, gcount;  // the group range; gcount = 0 when it lies outside the group table
  int32_t replicas, floor, ready_before;
  bool evaluated, available;
};

constexpr uint32_t kBudgetExcluded = LWSE_LOUT_BAD_TABLE | LWSE_LOUT_IRREGULAR | LWSE_LOUT_RUP_ERROR | LWSE_LOUT_STATUS_ERROR;

__device__ __forceinline__ int32_t clamp_i32(int64_t v) {
  return (int32_t)(v < INT32_MIN ? (int64_t)INT32_MIN : (v > INT32_MAX ? (int64_t)INT32_MAX : v));
}

// scaled_value (lwse_device.cuh) rounded down, kept in 64 bits as Go's int: the floor's mu must not wrap
// when a percentage above 100 of a large replicas passes int32.  (The sweep keeps its int32(mu), :313.)
__device__ __forceinline__ int64_t unavailable_i64(int32_t val, bool is_percent, int32_t total) {
  if (!is_percent) return val;
  const int64_t num = (int64_t)val * (int64_t)total;
  const int64_t q = num / 100;
  return (num - q * 100 != 0 && num < 0) ? q - 1 : q;
}

__device__ __forceinline__ LwsBudget budget_of(const lwse_lws_rec* lws, const lwse_lws_out* lws_out, uint32_t L,
                                               uint32_t n_groups) {
  const uint4* row = reinterpret_cast<const uint4*>(lws + L);
  const uint4 r0 = ldg_cached(row + 0), r1 = ldg_cached(row + 1), r3 = ldg_cached(row + 3);
  const uint4* orow = reinterpret_cast<const uint4*>(lws_out + L);
  const uint4 o0 = __ldg(orow + 0), o1 = __ldg(orow + 1);
  const uint32_t lflags = r0.w, oflags = o1.z;
  LwsBudget b;
  b.replicas = (int32_t)r1.x;
  b.gbase = r3.z;
  b.gcount = (uint64_t)r3.z + r3.w <= n_groups ? r3.w : 0u;
  b.evaluated = !(oflags & kBudgetExcluded) && !(lflags & LWSE_LWS_INTSTR_INVALID);
  b.available = ((oflags & LWSE_LOUT_COND_MASK) >> LWSE_LOUT_COND_SHIFT) == LWSE_COND_AVAILABLE;
  b.ready_before = (int32_t)o0.w;
  const int64_t mu = unavailable_i64((int32_t)r1.w, lflags & LWSE_LWS_UNAVAIL_IS_PERCENT, b.replicas);  // :302
  const int64_t fl = (int64_t)b.replicas - mu;
  b.floor = b.evaluated ? clamp_i32(fl < 0 ? 0 : fl) : 0;
  return b;
}

// The LWS row whose ready count revision-role row `row` takes under the link rule (the DS tick's linked_ready),
// or LWSE_NONE.  (lwse_ds_kernels.cu and lwse_ds_drain_wave_kernels.cu: the DS drain's definition in lwse.h.)
__device__ __forceinline__ uint32_t ds_link_target(const lwse_ds_link* links, const lwse_lws_rec* lws,
                                                   const lwse_lws_out* lws_out, uint32_t n_lws, uint32_t row, bool exists) {
  if (!exists) return LWSE_NONE;
  const uint4 l = ldg_stream(links + row);  // {uid lo, uid hi, lws_row, reserved}
  if (l.z >= n_lws) return LWSE_NONE;       // (LWSE_NONE included)
  const uint64_t uid = __ldg(reinterpret_cast<const unsigned long long*>(&lws[l.z].uid_hash));
  if (uid != u64_of(l.x, l.y)) return LWSE_NONE;
  constexpr uint32_t kNoUpdate = LWSE_LOUT_IRREGULAR | LWSE_LOUT_BAD_TABLE | LWSE_LOUT_RUP_ERROR | LWSE_LOUT_STATUS_ERROR;
  return (__ldg(&lws_out[l.z].flags) & kNoUpdate) ? LWSE_NONE : l.z;
}

}  // namespace lwse
