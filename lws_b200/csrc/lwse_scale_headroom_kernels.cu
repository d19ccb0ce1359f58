// Scale headroom (lwse_resident_scale_headroom, sm_90a); the definition is in lwse.h, the argument in DESIGN.md §3.5
// ("Scale headroom").  The setup is lwse_resident_rollout_place's chain on the resident rows: a settled entry's
// forecast peak is r0, so its row there is the probe at r0.  The clean R form an interval [r0, H], so each entry
// bisects (r0, hi) with its bounds in device memory, and one captured round replays for every bisection step.
//
//   scale_headroom_setup_kernel   a warp per entry (after the count kernel): the settled flags, R_pig, hi, |E| of
//                                 the largest probe; the entries that search, max |E|, sum |E|, the rounds.
//   per round, captured once and replayed:
//     scale_headroom_round_kernel a warp per entry: the probe R (the midpoint, or R_pig once the bisection ended
//                                 below it unprobed), its row started, |E(R)|, the entry, the item.
//     (launch_rollout_place pass 1: the scan, the fill, the rollout instance of place_ns_kernel, the finish)
//     scale_headroom_commit_kernel a thread per entry: lo or hi moved, the probe's row kept.
//   scale_headroom_finish_kernel  a thread per entry: the answer rows, the totals.
#include "lwse_device.cuh"
#include "lwse_launch.cuh"

namespace lwse {

// st[i].z: the LWSE_SHR_NOT_* bits, and
constexpr uint32_t kShrCeil = 1u << 8;    // hi is the ceiling c_i + 1 (not R_pig)
constexpr uint32_t kShrProbed = 1u << 9;  // hi has been probed: trig holds its row
constexpr uint32_t kShrSearch = 1u << 10; // settled, with a probe above r0 to make
constexpr uint32_t kShrNot = LWSE_SHR_NOT_EXCLUSIVE | LWSE_SHR_NOT_FORECAST | LWSE_SHR_NOT_SETTLED;

static unsigned warp_grid(uint64_t n, int sm_count) {  // a warp per entry, 8 warps per CTA
  uint64_t grid = (n + 7) / 8;
  if (grid < 1) grid = 1;
  const uint64_t cap = (uint64_t)sm_count * 8u;
  return (unsigned)(grid < cap ? grid : cap);
}

__device__ __forceinline__ bool shr_lacks_pod(const RolloutPlaceLaunch& p, uint32_t row) {
  return row < p.n_groups && !(__ldg(&p.groups[row].flags) & LWSE_GRP_POD_PRESENT);
}

// |E(R)| (warp-uniform): the groups below min(R, gc) without a leader pod, plus R - gc.
__device__ uint32_t shr_extra_count(const RolloutPlaceLaunch& p, uint32_t gb, uint32_t gc, uint32_t R) {
  const uint32_t lane = threadIdx.x & 31u, below = R < gc ? R : gc;
  uint32_t c = 0;
  for (uint32_t g = lane; g < below; g += 32u) c += shr_lacks_pod(p, gb + g) ? 1u : 0u;
  return __reduce_add_sync(0xFFFFFFFFu, c) + (R > gc ? R - gc : 0u);
}

// The smallest R with |E(R)| = t (warp-uniform).
__device__ uint32_t shr_pigeonhole(const RolloutPlaceLaunch& p, uint32_t gb, uint32_t gc, uint32_t t) {
  const uint32_t lane = threadIdx.x & 31u;
  uint32_t have = 0;
  for (uint32_t g0 = 0; g0 < gc; g0 += 32u) {
    const uint32_t g = g0 + lane;
    const uint32_t mask = __ballot_sync(0xFFFFFFFFu, g < gc && shr_lacks_pod(p, gb + g));
    const uint32_t k = (uint32_t)__popc(mask);
    if (have + k >= t) {  // the (t - have)-th missing group of this chunk is the t-th overall
      const bool hit = ((mask >> lane) & 1u) && (uint32_t)__popc(mask & ((2u << lane) - 1u)) == t - have;
      return g0 + (uint32_t)__ffs(__ballot_sync(0xFFFFFFFFu, hit));  // its index + 1
    }
    have += k;
  }
  return gc + (t - have);
}

__device__ __forceinline__ uint32_t shr_triggers(const uint32_t* row, uint32_t constraints) {
  return ((constraints & LWSE_RPW_STRANDED) && row[5]) || ((constraints & LWSE_RPW_BUMPED) && (row[6] || row[7]));
}

__device__ __forceinline__ uint32_t ceil_log2(uint32_t d) { return d > 1u ? 32u - (uint32_t)__clz(d - 1u) : 0u; }

// words: [0] entries that search [1] max |E| [2..3] sum |E| (u64) [4] rounds.
__global__ void __launch_bounds__(256) scale_headroom_setup_kernel(const ScaleHeadroomLaunch h) {
  const RolloutPlaceLaunch& p = h.p;
  const uint32_t lane = threadIdx.x & 31u, n_warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < p.n; i += n_warps) {
    const uint32_t L = __ldg(p.rows + i);
    const lwse_lws_rec& lr = p.lws[L];
    const lwse_lws_forecast& f = p.fc[L];
    const uint32_t lflags = __ldg(&lr.flags), fflags = __ldg(&f.flags);
    const int32_t r0 = __ldg(&lr.replicas);
    uint32_t bits = 0;
    if (!(lflags & LWSE_LWS_EXCLUSIVE_TOPOLOGY)) bits |= LWSE_SHR_NOT_EXCLUSIVE;
    if (fflags & (LWSE_LWSF_BAD_TABLE | LWSE_LWSF_NOT_FORECAST)) bits |= LWSE_SHR_NOT_FORECAST;
    if (!(lflags & LWSE_LWS_STS_EXISTS) || (lflags & LWSE_LWS_UPDATED) || r0 < 0 || __ldg(&lr.sts_replicas) != r0 ||
        __ldg(&lr.sts_partition) != 0 || __ldg(&lr.partition) != 0 ||
        (fflags & (LWSE_LWSF_ROLLING | LWSE_LWSF_UNFINISHED | LWSE_LWSF_HELD)) || __ldg(&f.peak_sts_replicas) != r0 ||
        __ldg(&f.final_replicas) != r0)
      bits |= LWSE_SHR_NOT_SETTLED;
    uint32_t hi = (uint32_t)r0 + 1u, m = 0, need = 0;
    if (bits == 0) {  // warp-uniform
      const uint32_t gb = __ldg(&lr.group_base), gc = __ldg(&lr.group_count);
      const uint32_t pig = shr_pigeonhole(p, gb, gc, h.n_domains + 1u);
      const int64_t c = h.ceilings ? (int64_t)__ldg(h.ceilings + i) : -1;
      if (c >= 0 && c + 1 <= (int64_t)pig) {
        bits |= kShrCeil;
        hi = (uint32_t)(c + 1);
      } else {
        hi = pig;
      }
      if (hi <= (uint32_t)r0) hi = (uint32_t)r0 + 1u;  // a ceiling below r0 (or R_pig <= r0: r0 strands)
      const uint32_t top = (bits & kShrCeil) ? hi - 1u : hi;  // the largest R a probe can take
      if (top > (uint32_t)r0) {
        bits |= kShrSearch;
        m = shr_extra_count(p, gb, gc, top);
        need = ceil_log2(hi - (uint32_t)r0) + ((bits & kShrCeil) ? 0u : 1u);
      }
    }
    if (lane != 0) continue;
    h.st[i] = make_uint4((uint32_t)r0, hi, bits, (uint32_t)r0);
    if (!(bits & kShrSearch)) continue;
    atomicAdd(h.words + 0, 1u);
    atomicMax(h.words + 1, m);
    atomicAdd(reinterpret_cast<unsigned long long*>(h.words + 2), (unsigned long long)m);
    atomicMax(h.words + 4, need);
  }
}

__global__ void __launch_bounds__(256) scale_headroom_round_kernel(const ScaleHeadroomLaunch h) {
  const RolloutPlaceLaunch& p = h.p;
  const uint32_t lane = threadIdx.x & 31u, n_warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < p.n; i += n_warps) {
    const uint4 s = __ldcg(h.st + i);
    uint32_t R = 0;
    if ((s.z & kShrSearch) && !shr_triggers(h.cur + (size_t)i * 16u, h.constraints)) {
      if (s.y - s.x > 1u) R = s.x + (s.y - s.x) / 2u;
      else if (!(s.z & (kShrCeil | kShrProbed))) R = s.y;  // the bisection ended below R_pig, never probed there
    }
    const uint32_t L = __ldg(p.rows + i);
    const uint32_t gb = __ldg(&p.lws[L].group_base), gc = __ldg(&p.lws[L].group_count);
    const uint32_t m = R ? shr_extra_count(p, gb, gc, R) : 0u;  // (R > r0 >= 0)
    if (lane != 0) continue;
    uint4* row = reinterpret_cast<uint4*>(p.rows_out + (size_t)i * 16u);
    row[0] = R ? make_uint4(LWSE_RPL_SOLVED, 0u, R, m) : make_uint4(0u, 0u, 0u, 0u);
    row[1] = row[2] = row[3] = make_uint4(0u, 0u, 0u, 0u);
    p.ent[i] = make_uint4(0u, m, gb, gc);
    p.e_count[i] = m;
    if (m) p.items[atomicAdd(p.counts + 0, 1u)] = make_uint2(i, __ldg(p.ns + i));
  }
}

__global__ void __launch_bounds__(256) scale_headroom_commit_kernel(const ScaleHeadroomLaunch h) {
  const RolloutPlaceLaunch& p = h.p;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += gridDim.x * blockDim.x) {
    const uint32_t* row = p.rows_out + (size_t)i * 16u;
    if (!(row[0] & LWSE_RPL_SOLVED)) continue;  // no probe this round
    uint4 s = __ldcg(h.st + i);
    uint32_t* keep;
    if (shr_triggers(row, h.constraints)) {
      s.y = row[2];
      s.z |= kShrProbed;
      keep = h.trig;
    } else {
      s.x = row[2];
      keep = h.clean;
    }
    h.st[i] = s;
    const uint4* src = reinterpret_cast<const uint4*>(row);
    uint4* dst = reinterpret_cast<uint4*>(keep + (size_t)i * 16u);
    for (uint32_t x = 0; x < 4; x++) dst[x] = src[x];
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) p.counts[0] = 0u;  // the next round's items
}

// out: [0] n_solved [1] n_blocked [2] n_at_ceiling [3] 0 [4..5] the headroom sum (u64), then n lwse_scale_headroom.
__global__ void __launch_bounds__(256) scale_headroom_finish_kernel(const ScaleHeadroomLaunch h) {
  const RolloutPlaceLaunch& p = h.p;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += gridDim.x * blockDim.x) {
    const uint4 s = __ldcg(h.st + i);
    const int32_t r0 = (int32_t)s.w;
    uint32_t* o = h.out + 8 + (size_t)i * 16u;
    for (uint32_t x = 4; x < 16; x++) o[x] = 0u;
    if (s.z & kShrNot) {
      o[0] = s.z & kShrNot;
      o[1] = (uint32_t)r0;
      o[2] = o[3] = 0xFFFFFFFFu;
      continue;
    }
    const uint32_t* cur = h.cur + (size_t)i * 16u;
    const uint32_t* src;
    uint32_t flags = LWSE_SHR_SOLVED;
    int32_t H, probe;
    if (shr_triggers(cur, h.constraints)) {
      flags |= LWSE_SHR_BLOCKED;
      H = -1;
      probe = r0;
      src = cur;
    } else if (s.z & kShrProbed) {
      H = (int32_t)s.x;
      probe = (int32_t)s.y;
      src = h.trig + (size_t)i * 16u;
    } else {  // hi is the ceiling, never probed: H = c_i (or r0 for a ceiling <= r0)
      flags |= LWSE_SHR_AT_CEILING;
      H = probe = (int32_t)s.x;
      src = H == r0 ? cur : h.clean + (size_t)i * 16u;
    }
    if (src[5]) flags |= LWSE_SHR_STRANDS;
    if (src[6] || src[7]) flags |= LWSE_SHR_BUMPS;
    o[0] = flags;
    o[1] = (uint32_t)r0;
    o[2] = (uint32_t)H;
    o[3] = (uint32_t)probe;
    for (uint32_t x = 0; x < 12; x++) o[4 + x] = src[3 + x];
    atomicAdd(h.out + 0, 1u);
    if (flags & LWSE_SHR_BLOCKED) atomicAdd(h.out + 1, 1u);
    if (flags & LWSE_SHR_AT_CEILING) atomicAdd(h.out + 2, 1u);
    if (H > r0) atomicAdd(reinterpret_cast<unsigned long long*>(h.out + 4), (unsigned long long)(H - r0));
  }
}

int launch_scale_headroom(const ScaleHeadroomLaunch* h, int pass, int sm_count, cudaStream_t s) {
  const unsigned grid = grid_for(h->p.n, 256, (uint32_t)sm_count * 4u);
  if (pass == 0) {
    scale_headroom_setup_kernel<<<warp_grid(h->p.n, sm_count), 256, 0, s>>>(*h);
    return launch_result(1);
  }
  if (pass == 1) {
    scale_headroom_round_kernel<<<warp_grid(h->p.n, sm_count), 256, 0, s>>>(*h);
    if (const int r = launch_result(0); r < 0) return r;
    const int solved = launch_rollout_place(&h->p, 1, sm_count, s);
    if (solved < 0) return solved;
    scale_headroom_commit_kernel<<<grid, 256, 0, s>>>(*h);
    return launch_result(solved + 2);
  }
  scale_headroom_finish_kernel<<<grid, 256, 0, s>>>(*h);
  return launch_result(1);
}

}  // namespace lwse
