// Rollout placement waves (lwse_resident_rollout_place_waves, sm_90a); the definition is in lwse.h, the argument in
// DESIGN.md §3.5 ("Rollout placement waves").  The setup is lwse_resident_rollout_place's chain; its rows are the
// alone rows.  Keys of different namespaces never wait for each other, so the plan runs in rounds: round r takes
// the r-th key of every namespace that has one.
//
//   rollout_waves_rank_kernel     one CTA: the key rows (status, alone), and per namespace, in query order, each
//                                 taking key's round; K_ns, T_ns, R, max T_ns and the active namespaces.
//   (place_index_scan_kernel)     K_ns -> ns_first.
//   rollout_waves_fill_kernel     a thread per key: the per-namespace key lists.
//   per round, captured once and replayed R times with the round in st[0]:
//     rollout_waves_items_kernel  a thread per active namespace: slot (ns, w) for every wave w < p_ns, an item
//                                 when the probe holds an extra row.
//     (place_ns_kernel, the wave instance)  one slot per item: the probe's diff into the slot's row.
//     rollout_waves_commit_kernel one CTA: per namespace the lowest clean column, else wave p_ns; the wave totals
//                                 take the new column's contribution in place of the old; the round advances.
//   rollout_waves_finish_kernel   one CTA: the wave rows (baseline totals added, namespaces per wave), the query
//                                 totals.
#include "lwse_device.cuh"
#include "lwse_launch.cuh"

namespace lwse {

constexpr uint32_t kWaveCounts = 11;  // placed, stranded, own_lost, bumped, then the seven what-if counters

__device__ __forceinline__ uint32_t* key_row(const RolloutPlaceWavesLaunch& w, uint32_t i) {
  return reinterpret_cast<uint32_t*>(w.out + 32) + (size_t)i * 4u;
}

__device__ __forceinline__ uint32_t alone_bits(const uint32_t* row) {  // a lwse_rollout_place row's verdicts
  return (row[5] ? LWSE_RPW_STRANDED : 0u) | ((row[6] || row[7]) ? LWSE_RPW_BUMPED : 0u);
}

// Keys in chunks of the CTA, in query order; within a chunk the warps take their turn, so that a namespace's
// rounds follow query order.
__global__ void __launch_bounds__(1024) rollout_waves_rank_kernel(const RolloutPlaceWavesLaunch w) {
  __shared__ uint32_t s_r, s_t, s_act;
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  const RolloutPlaceLaunch& p = w.p;
  if (tid == 0) s_r = s_t = s_act = 0u;
  __syncthreads();
  for (uint32_t base = 0; base < p.n; base += blockDim.x) {
    const uint32_t i = base + tid;
    bool part = false;
    uint32_t ns = LWSE_NONE, m = 0;
    if (i < p.n) {
      const uint32_t* row = p.rows_out + (size_t)i * 16u;
      const uint32_t alone = alone_bits(row);
      uint32_t status = LWSE_ROLLW_PLANNED;
      if (!(row[0] & LWSE_RPL_SOLVED)) {
        status = LWSE_ROLLW_NOT_SOLVED;
      } else if (alone & w.constraints) {
        status = LWSE_ROLLW_TRIGGERS_ALONE;
      } else {
        part = true;
        ns = __ldg(p.ns + i);
        m = row[3];
      }
      *reinterpret_cast<uint4*>(key_row(w, i)) = make_uint4(LWSE_NONE, status, (row[0] & LWSE_RPL_SOLVED) ? alone : 0u, 0u);
      w.rank[i] = LWSE_NONE;
    }
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, ns);
    const uint32_t leader = __ffs(peers) - 1u, below = (uint32_t)__popc(peers & ((1u << lane) - 1u));
    for (uint32_t t = 0; t < blockDim.x / 32u; t++) {
      if (warp == t) {
        uint32_t first = 0;
        if (part && lane == leader) {
          first = w.ns_count[ns];
          const uint32_t k = first + (uint32_t)__popc(peers);
          w.ns_count[ns] = k;
          atomicMax(&s_r, k);
          if (first == 0u) w.act[atomicAdd(&s_act, 1u)] = ns;
        }
        first = __shfl_sync(0xFFFFFFFFu, first, (int)leader);
        if (part) {
          w.rank[i] = first + below;
          atomicAdd(w.ns_extra + ns, m);
        }
      }
      __syncthreads();
    }
  }
  for (uint32_t a = tid; a < s_act; a += blockDim.x) atomicMax(&s_t, __ldcg(w.ns_extra + w.act[a]));
  __syncthreads();
  if (tid == 0) {
    w.st[2] = s_r;
    w.st[3] = s_t;
    w.st[4] = s_act;
  }
}

__global__ void __launch_bounds__(256) rollout_waves_fill_kernel(const RolloutPlaceWavesLaunch w) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < w.p.n; i += gridDim.x * blockDim.x) {
    const uint32_t r = __ldcg(w.rank + i);
    if (r != LWSE_NONE) w.ns_keys[__ldcg(w.ns_first + __ldg(w.p.ns + i)) + r] = i;
  }
}

__global__ void __launch_bounds__(256) rollout_waves_items_kernel(const RolloutPlaceWavesLaunch w) {
  const uint32_t r = __ldcg(w.st + 0), n_act = __ldcg(w.st + 4);
  for (uint32_t a = blockIdx.x * blockDim.x + threadIdx.x; a < n_act; a += gridDim.x * blockDim.x) {
    const uint32_t ns = __ldcg(w.act + a), f = __ldcg(w.ns_first + ns), K = __ldcg(w.ns_first + ns + 1u) - f;
    if (r >= K) continue;
    const uint32_t k = __ldcg(w.ns_keys + f + r), p = __ldcg(w.ns_open + ns), ek = __ldcg(&w.p.ent[k].y);
    for (uint32_t c = 0; c < p; c++) {
      const uint32_t slot = f + c, rows = __ldcg(w.col_rows + slot);
      uint4* res = reinterpret_cast<uint4*>(w.res + (size_t)slot * 16u);
      res[1] = res[2] = res[3] = make_uint4(0u, 0u, 0u, 0u);
      w.desc[slot] = make_uint4(k, f * w.wc + c * K, __ldcg(w.col_n + slot), rows);
      if (rows + ek) w.items[atomicAdd(w.st + 1, 1u)] = make_uint2(slot, ns);
    }
  }
}

// One CTA: the round's commits, then the round advances (nothing else reads st[0] or st[1] until the next round).
__global__ void __launch_bounds__(1024) rollout_waves_commit_kernel(const RolloutPlaceWavesLaunch w) {
  const RolloutPlaceLaunch& p = w.p;
  const uint32_t r = __ldcg(w.st + 0), n_act = __ldcg(w.st + 4);
  for (uint32_t a = threadIdx.x; a < n_act; a += blockDim.x) {
    const uint32_t ns = __ldcg(w.act + a), f = __ldcg(w.ns_first + ns), K = __ldcg(w.ns_first + ns + 1u) - f;
    if (r >= K) continue;
    const uint32_t k = __ldcg(w.ns_keys + f + r), p_ns = __ldcg(w.ns_open + ns);
    uint32_t wave = LWSE_NONE;
    for (uint32_t c = 0; c < p_ns && wave == LWSE_NONE; c++)
      if (!(alone_bits(w.res + (size_t)(f + c) * 16u) & w.constraints)) wave = c;
    uint32_t v[kWaveCounts];
    if (wave != LWSE_NONE) {
      for (uint32_t x = 0; x < kWaveCounts; x++) v[x] = __ldcg(w.res + (size_t)(f + wave) * 16u + 4u + x);
    } else if (p_ns < w.max_waves) {  // a new wave: the probe is {k} alone, the alone row (its totals as deltas)
      wave = p_ns;
      w.ns_open[ns] = p_ns + 1u;
      for (uint32_t x = 0; x < kWaveCounts; x++) v[x] = __ldcg(p.rows_out + (size_t)k * 16u + 4u + x);
      for (uint32_t x = 8; x < kWaveCounts; x++) v[x] -= __ldcg(p.counts + 20u + (x - 8u));
    } else {
      key_row(w, k)[1] = LWSE_ROLLW_NO_WAVE;
      continue;
    }
    const uint32_t slot = f + wave;
    uint32_t* old = w.contrib + (size_t)slot * kWaveCounts;
    for (uint32_t x = 0; x < kWaveCounts; x++) {
      if (v[x] != old[x]) atomicAdd(w.wtot + wave * 16u + 1u + x, v[x] - old[x]);
      old[x] = v[x];
    }
    atomicAdd(w.wtot + wave * 16u, 1u);
    const uint4 e = __ldcg(p.ent + k);
    const uint32_t n_list = w.col_n[slot], rows = w.col_rows[slot];
    w.col[(size_t)f * w.wc + (size_t)wave * K + n_list] = make_uint4(e.x, rows, e.z, e.w);
    w.col_n[slot] = n_list + 1u;
    w.col_rows[slot] = rows + e.y;
    key_row(w, k)[0] = wave;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    w.st[0] = r + 1u;
    w.st[1] = 0u;
  }
}

// out: [0] n_waves [1] n_planned [2] n_triggers_alone [3] n_no_wave [4] n_not_solved; then the keys; then the
// waves.
__global__ void __launch_bounds__(1024) rollout_waves_finish_kernel(const RolloutPlaceWavesLaunch w) {
  __shared__ uint32_t s_tot[5], s_ns[LWSE_DRAIN_WAVES_MAX];
  const uint32_t tid = threadIdx.x, n_act = __ldcg(w.st + 4);
  if (tid < 5) s_tot[tid] = 0u;
  if (tid < LWSE_DRAIN_WAVES_MAX) s_ns[tid] = 0u;
  __syncthreads();
  for (uint32_t a = tid; a < n_act; a += blockDim.x) {
    const uint32_t p_ns = __ldcg(w.ns_open + __ldcg(w.act + a));
    atomicMax(&s_tot[0], p_ns);
    for (uint32_t c = 0; c < p_ns; c++) atomicAdd(&s_ns[c], 1u);
  }
  for (uint32_t i = tid; i < w.p.n; i += blockDim.x) {
    const uint32_t st = key_row(w, i)[1];
    atomicAdd(&s_tot[st == LWSE_ROLLW_PLANNED ? 1 : st == LWSE_ROLLW_TRIGGERS_ALONE ? 2 : st == LWSE_ROLLW_NO_WAVE ? 3 : 4], 1u);
  }
  __syncthreads();
  uint32_t* tot = reinterpret_cast<uint32_t*>(w.out);
  if (tid < 5) tot[tid] = s_tot[tid];
  if (tid < s_tot[0]) {  // lwse_rollout_wave
    const uint32_t* t = w.wtot + tid * 16u;
    uint32_t* o = reinterpret_cast<uint32_t*>(w.out + 32 + (size_t)w.p.n * 16u) + tid * 16u;
    o[0] = t[0];
    o[1] = t[1] + t[2];  // surge: placed + stranded
    for (uint32_t x = 0; x < kWaveCounts; x++) o[2 + x] = t[1 + x] + (x >= 8 ? __ldcg(w.p.counts + 20u + (x - 8u)) : 0u);
    o[13] = s_ns[tid];
    o[14] = o[15] = 0u;
  }
}

int launch_rollout_place_waves(const RolloutPlaceWavesLaunch* w, int pass, int sm_count, cudaStream_t s) {
  const unsigned grid = grid_for(w->p.n, 256, (uint32_t)sm_count * 4u);
  if (pass == 0) {
    rollout_waves_rank_kernel<<<1, 1024, 0, s>>>(*w);
    if (const int r = launch_result(0); r < 0) return r;
    if (const int r = launch_index_scan(w->ns_count, w->ns_first, w->ns_cursor, w->p.n_namespaces, s); r < 0) return r;
    rollout_waves_fill_kernel<<<grid, 256, 0, s>>>(*w);
    return launch_result(3);
  }
  if (pass == 1) {
    rollout_waves_items_kernel<<<grid, 256, 0, s>>>(*w);
    if (const int r = launch_result(0); r < 0) return r;
    int n = 1;
    if (w->grid) {
      if (const int r = launch_place_ns_rollout_wave(w, s); r < 0) return r;
      n++;
    }
    rollout_waves_commit_kernel<<<1, 1024, 0, s>>>(*w);
    return launch_result(n + 1);
  }
  rollout_waves_finish_kernel<<<1, 1024, 0, s>>>(*w);
  return launch_result(1);
}

}  // namespace lwse
