// Rollout what-if of LeaderWorkerSets (lwse_resident_rollout_whatif, sm_90a); the definition is in lwse.h.
//
//   scan (three kernels)             the group_count of each proposal's resident row → its offset into
//                                    the scratch group table, and the total (lwse_device.cuh)
//   rollout_whatif_gather_kernel     one warp per proposal: the scratch proposal row's range, and a copy
//                                    of the resident range's group rows, owned rows pointing at the
//                                    scratch row, foreign-owned rows recorded
//   rollout_whatif_restore_kernel    after the group pass: the foreign-owned rows get the resident sweep's
//                                    result back, in group_out and in the sweep's flag column
// The engine runs the sweep's group pass between the gather and the restore, and its LWS pass and the
// forecast after the restore.
#include "lwse_device.cuh"
#include "lwse_launch.cuh"

namespace lwse {

// The layout: counts → exclusive offsets (launch_forecast_scan).  A proposal gathers the group_count of
// its resident row, or nothing when that row's range lies outside the resident group table.
struct WhatifLayoutOp {
  const lwse_lws_rec* lws;
  const uint32_t* rows;
  uint32_t n_groups;
  unsigned long long* off;
  __device__ __forceinline__ unsigned long long count(uint32_t i) const {
    const uint4 r3 = ldg_stream(reinterpret_cast<const uint4*>(lws + __ldg(rows + i)) + 3);
    return (uint64_t)r3.z + r3.w <= n_groups ? r3.w : 0u;
  }
  __device__ __forceinline__ unsigned long long apply(uint32_t i, unsigned long long base, unsigned long long) const {
    off[i] = base;
    return 0ull;
  }
};

__global__ void __launch_bounds__(256) rollout_whatif_gather_kernel(const RolloutWhatifHost a) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t n_warps = gridDim.x * (blockDim.x >> 5);
  for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < a.n; i += n_warps) {
    const uint32_t L = __ldg(a.rows + i);
    const uint4 r3 = ldg_stream(reinterpret_cast<const uint4*>(a.lws + L) + 3);
    const uint32_t gbase = r3.z;
    const bool in_table = (uint64_t)r3.z + r3.w <= a.n_groups;
    const uint32_t gc = in_table ? r3.w : 0u;
    const uint32_t base = (uint32_t)a.off[i];  // < 2^32: the engine refuses a larger gather
    if (lane == 0) {
      // the caller's row with the resident range; a range outside the table stays outside the scratch
      // table (base 0xFFFFFFFF), so that the LWS pass and the forecast report it as the sweep does
      uint4* w3 = reinterpret_cast<uint4*>(a.s_lws + i) + 3;
      uint4 v = *w3;
      v.z = in_table ? base : 0xFFFFFFFFu;
      v.w = r3.w;
      *w3 = v;
    }
    const uint4* src = reinterpret_cast<const uint4*>(a.groups + gbase);
    uint4* dst = reinterpret_cast<uint4*>(a.s_groups + base);
    const uint64_t n_words = (uint64_t)gc * 4u;  // 64-byte rows: four 16-byte words each
    for (uint64_t k = lane; k < n_words; k += 32u) {
      uint4 v = ldg_stream(src + k);
      if ((k & 3u) == 3u) {  // {lws_index, ..}
        const uint32_t r = (uint32_t)(k >> 2);
        const bool own = v.x == L;
        a.s_src[base + r] = own ? LWSE_NONE : gbase + r;
        v.x = own ? i : LWSE_NONE;  // a foreign row's result comes back in the restore
      }
      dst[k] = v;
    }
  }
}

__global__ void __launch_bounds__(256) rollout_whatif_restore_kernel(const uint32_t* __restrict__ src,
                                                                     const lwse_group_out* __restrict__ baseline,
                                                                     lwse_group_out* __restrict__ out,
                                                                     uint8_t* __restrict__ gflag8, uint32_t n_rows) {
  for (uint32_t g = blockIdx.x * blockDim.x + threadIdx.x; g < n_rows; g += gridDim.x * blockDim.x) {
    const uint32_t r = __ldg(src + g);
    if (r == LWSE_NONE) continue;
    const uint4 v = ldg_stream(reinterpret_cast<const uint4*>(baseline + r));
    reinterpret_cast<uint4*>(out)[g] = v;
    gflag8[g] = (uint8_t)(v.x & 0x1Fu);  // the low five bits the LWS pass reads (lwse_lws_kernels.cu)
  }
}

int launch_rollout_whatif_layout(const RolloutWhatifHost* h, unsigned long long* sums, unsigned long long* total,
                                 cudaStream_t s) {
  launch_forecast_scan(WhatifLayoutOp{h->lws, h->rows, h->n_groups, h->off}, h->n, sums, total, nullptr, s);
  return launch_result(h->n ? 3 : 1);
}

int launch_rollout_whatif_gather(const RolloutWhatifHost* h, int sm_count, cudaStream_t s) {
  if (h->n == 0) return 0;
  const uint32_t want = (h->n + 7u) / 8u, cap = (uint32_t)sm_count * 8u;
  rollout_whatif_gather_kernel<<<want < cap ? want : cap, 256, 0, s>>>(*h);
  return launch_result(1);
}

int launch_rollout_whatif_restore(const uint32_t* d_src, const lwse_group_out* d_baseline, lwse_group_out* d_out,
                                  uint8_t* d_gflag8, uint32_t n_rows, int sm_count, cudaStream_t s) {
  if (n_rows == 0) return 0;
  const uint32_t want = (n_rows + 255u) / 256u, cap = (uint32_t)sm_count * 8u;
  rollout_whatif_restore_kernel<<<want < cap ? want : cap, 256, 0, s>>>(d_src, d_baseline, d_out, d_gflag8, n_rows);
  return launch_result(1);
}

}  // namespace lwse
