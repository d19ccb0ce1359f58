// Rollout placement (lwse_resident_rollout_place, sm_90a); the definition is in lwse.h, the argument in DESIGN.md
// §3.5 ("Rollout placement").
//
//   rollout_place_count_kernel   a warp per entry: the flags, |E_i| (the groups below min(peak, group_count) without a
//                                leader pod, plus peak - group_count), the entry's row started, the items.
//   (place_index_scan_kernel)    |E_i| -> each entry's first extra row.
//   rollout_place_fill_kernel    a warp per entry: E_i's rows in ascending group index, with the encoder's mix.
//   (place_ns_kernel, the rollout instance)   one namespace per item, its diff into the entry's row.
//   rollout_place_finish_kernel  a thread per entry: the baseline totals added, STRANDS / BUMPS, the query totals.
#include "lwse_device.cuh"
#include "lwse_launch.cuh"

namespace lwse {

static unsigned warp_grid(uint64_t n, int sm_count) {  // a warp per entry, 8 warps per CTA
  uint64_t grid = (n + 7) / 8;
  if (grid < 1) grid = 1;
  const uint64_t cap = (uint64_t)sm_count * 8u;
  return (unsigned)(grid < cap ? grid : cap);
}

__device__ __forceinline__ const lwse_lws_rec& proposal_of(const RolloutPlaceLaunch& p, uint32_t i) {
  return p.recs ? p.recs[i] : p.lws[p.rows[i]];
}

// encode_place_requests' priority and key mix of (uid_hash, group index)
__device__ __forceinline__ void encoder_mix(uint64_t uid, uint64_t g, uint64_t* priority, uint64_t* key) {
  uint64_t pr = (uid ^ (g * 0x9E3779B97F4A7C15ull)) * 0xBF58476D1CE4E5B9ull;
  pr ^= pr >> 31;
  uint64_t k = (uid + g) * 0x94D049BB133111EBull;
  k ^= k >> 29;
  *priority = pr;
  *key = k;
}

__device__ __forceinline__ bool lacks_pod(const RolloutPlaceLaunch& p, uint32_t row) {
  return row < p.n_groups && !(__ldg(&p.groups[row].flags) & LWSE_GRP_POD_PRESENT);
}

__global__ void __launch_bounds__(256) rollout_place_count_kernel(const RolloutPlaceLaunch p) {
  const uint32_t lane = threadIdx.x & 31u, n_warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < p.n; i += n_warps) {
    const uint32_t L = __ldg(p.rows + i);
    const lwse_lws_rec& lr = p.lws[L];
    const lwse_lws_rec& pr = proposal_of(p, i);
    const lwse_lws_forecast& f = p.fc[p.fc_by_row ? L : i];
    const uint32_t lflags = __ldg(&lr.flags), fflags = __ldg(&f.flags);
    const int32_t peak_raw = __ldg(&f.peak_sts_replicas);
    const uint32_t peak = peak_raw > 0 ? (uint32_t)peak_raw : 0u;
    const uint32_t gb = __ldg(&lr.group_base), gc = __ldg(&lr.group_count);
    uint32_t flags = 0;
    if (!(lflags & LWSE_LWS_EXCLUSIVE_TOPOLOGY)) flags |= LWSE_RPL_NOT_EXCLUSIVE;
    if (fflags & (LWSE_LWSF_BAD_TABLE | LWSE_LWSF_NOT_FORECAST)) flags |= LWSE_RPL_NOT_FORECAST;
    if (__ldg(&pr.size) != __ldg(&lr.size) || ((__ldg(&pr.flags) ^ lflags) & LWSE_LWS_EXCLUSIVE_TOPOLOGY))
      flags |= LWSE_RPL_NOT_MODELLED;
    uint64_t m = 0;
    if (flags == 0) {  // warp-uniform
      const uint32_t below = peak < gc ? peak : gc;
      uint32_t c = 0;
      for (uint32_t g = lane; g < below; g += 32u) c += lacks_pod(p, gb + g) ? 1u : 0u;
      m = (uint64_t)__reduce_add_sync(0xFFFFFFFFu, c) + (peak > gc ? peak - gc : 0u);
      flags = LWSE_RPL_SOLVED;
    }
    if (lane != 0) continue;
    const uint32_t m32 = m < 0xFFFFFFFFull ? (uint32_t)m : 0xFFFFFFFFu;
    uint4* row = reinterpret_cast<uint4*>(p.rows_out + (size_t)i * 16u);
    row[0] = make_uint4(flags, fflags, (uint32_t)peak_raw, m32);
    row[1] = make_uint4(0u, 0u, 0u, 0u);
    row[2] = make_uint4(0u, 0u, 0u, 0u);
    row[3] = make_uint4(0u, 0u, 0u, 0u);
    p.ent[i] = make_uint4(0u, m32, gb, gc);
    p.e_count[i] = m32;
    if (m == 0) continue;
    p.items[atomicAdd(p.counts + 0, 1u)] = make_uint2(i, __ldg(p.ns + i));
    atomicMax(p.counts + 1, m32);
    atomicAdd(reinterpret_cast<unsigned long long*>(p.counts + 2), (unsigned long long)m);
  }
}

// After the scan (e_first) and the host's check that every |E_i| fits the 24-bit row keys.
__global__ void __launch_bounds__(256) rollout_place_fill_kernel(const RolloutPlaceLaunch p) {
  const uint32_t lane = threadIdx.x & 31u, n_warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < p.n; i += n_warps) {
    const uint4 ent = __ldcg(p.ent + i);
    if (ent.y == 0u) continue;  // warp-uniform
    const uint32_t first = __ldcg(p.e_first + i);
    if (lane == 0) p.ent[i].x = first;
    const lwse_lws_rec& pr = proposal_of(p, i);
    const uint64_t uid = pr.uid_hash;
    const int32_t size = pr.size;
    const uint32_t ns = __ldg(p.ns + i), gb = ent.z, gc = ent.w;
    const uint32_t peak = (uint32_t)__ldcg(reinterpret_cast<const int32_t*>(p.rows_out + (size_t)i * 16u) + 2);
    auto put = [&](uint32_t j, uint32_t g) {
      lwse_place_req q;
      encoder_mix(uid, g, &q.priority, &q.group_key);
      q.group = gb + g;
      q.ns = ns;
      q.size = size;
      q.leader_node = LWSE_NONE;
      p.extra[first + j] = q;
    };
    const uint32_t below = peak < gc ? peak : gc;
    uint32_t at = 0;  // E_i's rows so far
    for (uint32_t g0 = 0; g0 < below; g0 += 32u) {
      const uint32_t g = g0 + lane;
      const bool extra = g < below && lacks_pod(p, gb + g);
      const uint32_t mask = __ballot_sync(0xFFFFFFFFu, extra);
      if (extra) put(at + (uint32_t)__popc(mask & ((1u << lane) - 1u)), g);
      at += (uint32_t)__popc(mask);
    }
    for (uint32_t t = lane; gc + t < peak; t += 32u) put(at + t, gc + t);
  }
}

// counts: [4] entries solved [5] entries that strand [6..7] surge rows (u64) [8..9] stranded rows (u64); the baseline's
// PLACED / UNSCHEDULABLE / CONFLICT at [20..22].
__global__ void __launch_bounds__(256) rollout_place_finish_kernel(const RolloutPlaceLaunch p) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += gridDim.x * blockDim.x) {
    uint32_t* row = p.rows_out + (size_t)i * 16u;
    uint32_t flags = row[0];
    if (!(flags & LWSE_RPL_SOLVED)) continue;
    row[12] += __ldcg(p.counts + 20);
    row[13] += __ldcg(p.counts + 21);
    row[14] += __ldcg(p.counts + 22);
    if (row[5]) flags |= LWSE_RPL_STRANDS;
    if (row[7]) flags |= LWSE_RPL_BUMPS;
    row[0] = flags;
    atomicAdd(p.counts + 4, 1u);
    if (row[5]) atomicAdd(p.counts + 5, 1u);
    if (row[3]) atomicAdd(reinterpret_cast<unsigned long long*>(p.counts + 6), (unsigned long long)row[3]);
    if (row[5]) atomicAdd(reinterpret_cast<unsigned long long*>(p.counts + 8), (unsigned long long)row[5]);
  }
}

int launch_rollout_place(const RolloutPlaceLaunch* p, int pass, int sm_count, cudaStream_t s) {
  if (pass == 0) {
    rollout_place_count_kernel<<<warp_grid(p->n, sm_count), 256, 0, s>>>(*p);
    return launch_result(1);
  }
  int n = 0;
  if (const int r = launch_index_scan(p->e_count, p->e_first, p->e_cursor, p->n, s); r < 0) return r;
  rollout_place_fill_kernel<<<warp_grid(p->n, sm_count), 256, 0, s>>>(*p);
  if (const int r = launch_result(0); r < 0) return r;
  n = 2;
  if (p->grid) {
    const int solved = launch_place_ns_rollout(p, sm_count, s);
    if (solved < 0) return solved;
    n += solved;
  }
  rollout_place_finish_kernel<<<grid_for(p->n, 256, (uint32_t)sm_count * 4u), 256, 0, s>>>(*p);
  return launch_result(n + 1);
}

}  // namespace lwse
