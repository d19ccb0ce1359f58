// Drain waves (lwse_resident_drain_waves, sm_90a); the definition is in lwse.h, the argument in DESIGN.md §3.5.
//
// After the drain budget's pass 0 (the key rows) and its pair walk (every restart pair key << 32 | group):
//   drain_waves_keys_kernel    a thread per listed key: its position, its bucket size (the key row's
//                              groups_restarted: one per pair) and the alone columns of its output row; the
//                              pair total over every key, which sizes the pair list.
//   drain_waves_fill_kernel    a thread per pair: the pairs of listed keys into their key's bucket (by cursor, after
//                              the scan), each with its owner LWS row (member or not), its baseline ready bit, its
//                              below-replicas bit and its pod_count; the touched LWS rows marked.
//   drain_waves_dense_kernel   the touched LWS rows compacted (after their scan): each dense row's ready_before,
//                              floor and flags, and every pair's owner mapped to its dense row.
//   drain_waves_plan_kernel    one CTA walks the keys in order.  Per key, over (pair, wave) items: the ready
//                              pairs of evaluated rows are added to the lost counters of every open wave that does
//                              not hold their group yet and of the next wave (the key alone); the counters are
//                              checked against the rows' slack; the first feasible wave is taken; the other
//                              columns are taken back and the key's groups join the wave it took.
//   drain_waves_finish_kernel  every dense row's waves into their lws_touched / lws_loses_available / min_margin,
//                              and every planned key's pods and leaders into its wave.
// The DS drain waves (lwse_resident_ds_drain_waves) run the fill, dense and plan bodies with kCapped: pairs of linked
// rows are bound too, and each dense row carries the slack its DS caps and the caller's constraints give it.
#include "lwse_device.cuh"
#include "lwse_launch.cuh"

namespace lwse {

// A pair record: {group, owner (the LWS row, then its dense row; LWSE_NONE: not a member), bits, pod_count}.
constexpr uint32_t kPairMember = 1u << 0;
constexpr uint32_t kPairReady = 1u << 1;    // the group's baseline row has COND_READY
constexpr uint32_t kPairReadyNb = 1u << 2;  // ready, and its index in the LWS row's range is below replicas
constexpr uint32_t kPairBound = 1u << 3;    // ready, of a member group of an evaluated row: it counts against a floor
                                            // (the DS plan: of an evaluated or a linked row)
constexpr uint32_t kDenseEvaluated = 1u << 0, kDenseAvailable = 1u << 1;
constexpr uint32_t kDenseCapped = 1u << 2;  // the DS plan: some constraint bounds the row, its slack in w

// (pair, wave) items the plan kernel takes per pass: a key's pairs times the open waves plus one.
constexpr uint32_t kPlanThreads = 512;

__global__ void __launch_bounds__(256) drain_waves_keys_kernel(const DrainWavesLaunch p) {
  const uint32_t stride = gridDim.x * blockDim.x;
  unsigned long long pairs = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < p.m || i < p.n_keys; i += stride) {
    if (i < p.n_keys) pairs += __ldg(&p.cost[i].groups_restarted);
    if (i >= p.m) continue;
    const uint32_t key = __ldg(p.ids + i);
    const lwse_drain_budget_cost* c = p.cost + key;
    const uint32_t groups = __ldg(&c->groups_restarted);
    p.pos_of[key] = i;
    p.count[i] = groups;
    uint4* row = reinterpret_cast<uint4*>(p.out + 16 + (size_t)i * sizeof(lwse_drain_wave_key));
    row[0] = make_uint4(key, LWSE_NONE, LWSE_DRAINW_NO_WAVE, groups);
    row[1] = make_uint4(__ldg(&c->ready_restarted), 0u, 0u, 0u);
  }
  for (int off = 16; off > 0; off >>= 1) pairs += __shfl_xor_sync(0xFFFFFFFFu, pairs, off);
  if ((threadIdx.x & 31u) == 0 && pairs) atomicAdd(p.counts, pairs);
}

// kCapped (the DS plan): a ready member pair is also bound when some revision-role row a DS sweep reads takes the
// value of its LWS row (caps[L] has kCapLinked), evaluated or not.
template <bool kCapped>
__device__ __forceinline__ void drain_waves_fill(const DrainWavesLaunch& p, const uint32_t* caps) {
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < p.n_pairs; j += gridDim.x * blockDim.x) {
    const unsigned long long pr = __ldg(p.pairs + j);
    const uint32_t key = (uint32_t)(pr >> 32), g = (uint32_t)pr;
    const uint32_t pos = key < p.n_keys ? __ldcg(p.pos_of + key) : LWSE_NONE;
    if (pos == LWSE_NONE) continue;  // a key the query does not list
    const uint4 cc = __ldg(reinterpret_cast<const uint4*>(p.groups + g) + 2), cd = __ldg(reinterpret_cast<const uint4*>(p.groups + g) + 3);
    const uint32_t pod_count = cc.w, L = cd.x;  // (the walk emits only groups with lws_index < n_lws)
    const uint4 l1 = ldg_cached(reinterpret_cast<const uint4*>(p.lws + L) + 1), l3 = ldg_cached(reinterpret_cast<const uint4*>(p.lws + L) + 3);
    const uint32_t index = g - l3.z;
    const bool member = (uint64_t)l3.z + l3.w <= p.n_groups && g >= l3.z && index < l3.w;
    const bool ready = (__ldg(&p.baseline[g].flags) & LWSE_GOUT_COND_READY) != 0u;
    uint32_t bits = ready ? kPairReady : 0u;
    if (member) {
      bits |= kPairMember;
      if (ready && (int64_t)index < (int64_t)(int32_t)l1.x) bits |= kPairReadyNb;
      if constexpr (kCapped) {
        if (ready && ((__ldg(caps + L) & kCapLinked) || budget_of(p.lws, p.lws_out, L, p.n_groups).evaluated)) bits |= kPairBound;
      } else {
        if (ready && budget_of(p.lws, p.lws_out, L, p.n_groups).evaluated) bits |= kPairBound;
      }
      p.l_count[L] = 1u;
    }
    const uint32_t at = atomicAdd(p.cursor + pos, 1u);
    if (at < __ldcg(p.first + pos + 1u)) p.recs[at] = make_uint4(g, member ? L : LWSE_NONE, bits, pod_count);
    else atomicAdd(p.counts + 1, 1ull);  // more pairs than the key row counted: the call fails
  }
}

__global__ void __launch_bounds__(256) drain_waves_fill_kernel(const DrainWavesLaunch p) { drain_waves_fill<false>(p, nullptr); }

// kCapped: the dense row's w holds the row's slack under `constraints` (lwse.h, "DS drain waves"), clamped to
// int32, and kDenseCapped is set when some constraint bounds the row.  The clamp keeps every answer: a bound
// counter is >= 1 where it is checked, and the minimum is at most ready_before - 1 or ready_before - floor.
template <bool kCapped>
__device__ __forceinline__ void drain_waves_dense(const DrainWavesLaunch& p, const uint32_t* caps, uint32_t constraints) {
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t n_listed = __ldcg(p.first + p.m);
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < p.n_lws || i < n_listed; i += stride) {
    if (i < p.n_lws) {
      const uint32_t d = __ldcg(p.l_first + i);
      if (__ldcg(p.l_first + i + 1) != d) {
        const LwsBudget b = budget_of(p.lws, p.lws_out, i, p.n_groups);
        uint32_t flags = (b.evaluated ? kDenseEvaluated : 0u) | (b.available ? kDenseAvailable : 0u), slack = 0u;
        if constexpr (kCapped) {
          const uint32_t c = __ldg(caps + i) & constraints;
          int64_t cap = INT64_MAX;
          if ((constraints & LWSE_DSW_LWS_FLOOR) && b.evaluated) cap = (int64_t)b.ready_before - b.floor;
          if (c & (LWSE_DSW_DS_SERVICE | LWSE_DSW_DS_OLD_SERVICE)) cap = min(cap, (int64_t)b.ready_before - 1);
          if (c & LWSE_DSW_DS_STALL) cap = min(cap, (int64_t)0);
          if (cap != INT64_MAX) {
            flags |= kDenseCapped;
            slack = (uint32_t)clamp_i32(cap);
          }
        }
        p.dense[d] = make_uint4((uint32_t)b.ready_before, (uint32_t)b.floor, flags, slack);
      }
    }
    if (i < n_listed) {
      const uint32_t L = p.recs[i].y;
      if (L != LWSE_NONE) p.recs[i].y = __ldcg(p.l_first + L);
    }
  }
}

__global__ void __launch_bounds__(256) drain_waves_dense_kernel(const DrainWavesLaunch p) { drain_waves_dense<false>(p, nullptr, 0u); }

template <bool kCapped>
__device__ __forceinline__ int64_t slack_of(const uint4 d) {
  if constexpr (kCapped) return (d.z & kDenseCapped) ? (int64_t)(int32_t)d.w : INT64_MAX;
  return (int64_t)(int32_t)d.x - (int32_t)d.y;
}

template <bool kCapped>
__device__ __forceinline__ void drain_waves_plan(const DrainWavesLaunch& p) {
  __shared__ unsigned long long s_bad, s_recreated[LWSE_DRAIN_WAVES_MAX];
  __shared__ uint32_t s_groups[LWSE_DRAIN_WAVES_MAX], s_ready[LWSE_DRAIN_WAVES_MAX], s_keys[LWSE_DRAIN_WAVES_MAX];
  __shared__ uint32_t s_alone_bad, s_touched, s_breached, s_wave, s_open, s_status[3];
  const uint32_t tid = threadIdx.x;
  if (tid < LWSE_DRAIN_WAVES_MAX) {
    s_recreated[tid] = 0ull;
    s_groups[tid] = s_ready[tid] = s_keys[tid] = 0u;
  }
  if (tid == 0) {
    s_bad = 0ull;
    s_alone_bad = s_touched = s_breached = s_open = 0u;
    s_status[0] = s_status[1] = s_status[2] = 0u;
  }
  __syncthreads();
  uint32_t n_open = 0, b = 0;
  for (uint32_t i = 0; i < p.m; i++) {
    const uint32_t e = __ldg(p.first + i + 1);
    const uint32_t cols = n_open + 1;  // the open waves, and the next one: the key alone
    const uint32_t items = (e - b) * cols;
    // 1. add: every bound pair to the lost counter of each column that does not hold its group yet
    for (uint32_t j = tid; j < items; j += kPlanThreads) {
      const uint4 r = __ldg(p.recs + b + j / cols);
      const uint32_t w = j % cols;
      if (w == 0 && (r.z & kPairMember) && atomicExch(p.stamps + 2u * r.y, i + 1u) != i + 1u) atomicAdd(&s_touched, 1u);
      if ((r.z & kPairBound) && (w == n_open || !((__ldcg(p.g_waves + r.x) >> w) & 1ull)))
        atomicAdd(p.lost + (size_t)r.y * p.cols + w, 1u);
    }
    __syncthreads();
    // 2. check: a column whose counter passes the row's slack cannot take the key
    for (uint32_t j = tid; j < items; j += kPlanThreads) {
      const uint4 r = __ldg(p.recs + b + j / cols);
      const uint32_t w = j % cols;
      if (!(r.z & kPairBound) || !(w == n_open || !((__ldcg(p.g_waves + r.x) >> w) & 1ull))) continue;
      if ((int64_t)__ldcg(p.lost + (size_t)r.y * p.cols + w) <= slack_of<kCapped>(__ldg(p.dense + r.y))) continue;
      if (w < n_open) {
        atomicOr(&s_bad, 1ull << w);
      } else {
        s_alone_bad = 1u;
        if (atomicExch(p.stamps + 2u * r.y + 1u, i + 1u) != i + 1u) atomicAdd(&s_breached, 1u);
      }
    }
    __syncthreads();
    // 3. the first of BREACHES_ALONE, the lowest feasible open wave, a new wave, NO_WAVE
    if (tid == 0) {
      uint32_t wave = LWSE_NONE, status = LWSE_DRAINW_BREACHES_ALONE;
      if (!s_alone_bad) {
        const unsigned long long open = n_open >= 64u ? ~0ull : (1ull << n_open) - 1ull;
        const unsigned long long ok = open & ~s_bad;
        status = LWSE_DRAINW_PLANNED;
        if (ok) {
          wave = (uint32_t)(__ffsll((long long)ok) - 1);
        } else if (n_open < p.max_waves) {
          wave = n_open;
          s_open = n_open + 1u;
        } else {
          status = LWSE_DRAINW_NO_WAVE;
        }
      }
      if (wave != LWSE_NONE) s_keys[wave]++;
      s_status[status]++;
      uint32_t* row = reinterpret_cast<uint32_t*>(p.out + 16 + (size_t)i * sizeof(lwse_drain_wave_key));
      row[1] = wave;
      row[2] = status;
      row[5] = s_touched;
      row[6] = s_breached;
      s_wave = wave;
      s_bad = 0ull;
      s_alone_bad = s_touched = s_breached = 0u;
    }
    __syncthreads();
    // 4. the other columns taken back; the key's groups join its wave
    const uint32_t wave = s_wave;
    for (uint32_t j = tid; j < items; j += kPlanThreads) {
      const uint4 r = __ldg(p.recs + b + j / cols);
      const uint32_t w = j % cols;
      if (w != wave) {
        if ((r.z & kPairBound) && (w == n_open || !((__ldcg(p.g_waves + r.x) >> w) & 1ull)))
          atomicSub(p.lost + (size_t)r.y * p.cols + w, 1u);
        continue;
      }
      const unsigned long long bit = 1ull << w;
      if (!(atomicOr(p.g_waves + r.x, bit) & bit)) {  // the group's first pair in this wave
        atomicAdd(&s_groups[w], 1u);
        if (r.z & kPairReady) atomicAdd(&s_ready[w], 1u);
        atomicAdd(&s_recreated[w], (unsigned long long)r.w);
      }
      if (r.z & kPairMember) {
        atomicOr(p.row_waves + 2u * r.y, bit);
        if (r.z & kPairReadyNb) atomicOr(p.row_waves + 2u * r.y + 1u, bit);
      }
    }
    n_open = s_open;
    b = e;
    __syncthreads();
  }
  uint8_t* waves = p.out + 16 + (size_t)p.m * sizeof(lwse_drain_wave_key);
  if (tid < n_open) {
    uint4* row = reinterpret_cast<uint4*>(waves + (size_t)tid * sizeof(lwse_drain_wave));
    row[0] = make_uint4(s_keys[tid], 0u, 0u, 0u);
    row[1] = make_uint4(0u, s_groups[tid], s_ready[tid], (uint32_t)INT32_MAX);
    row[2] = make_uint4((uint32_t)s_recreated[tid], (uint32_t)(s_recreated[tid] >> 32), 0u, 0u);
  }
  if (tid == 0)
    *reinterpret_cast<uint4*>(p.out) = make_uint4(n_open, s_status[LWSE_DRAINW_PLANNED], s_status[LWSE_DRAINW_BREACHES_ALONE],
                                                  s_status[LWSE_DRAINW_NO_WAVE]);
}

__global__ void __launch_bounds__(kPlanThreads, 1) drain_waves_plan_kernel(const DrainWavesLaunch p) { drain_waves_plan<false>(p); }

__global__ void __launch_bounds__(256) drain_waves_finish_kernel(const DrainWavesLaunch p) {
  lwse_drain_wave* waves = reinterpret_cast<lwse_drain_wave*>(p.out + 16 + (size_t)p.m * sizeof(lwse_drain_wave_key));
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < p.n_dense || i < p.m; i += stride) {
    if (i < p.n_dense) {
      unsigned long long t = p.row_waves[2u * i];
      const unsigned long long nb = p.row_waves[2u * i + 1u];
      const uint4 d = __ldg(p.dense + i);
      while (t) {
        const uint32_t w = (uint32_t)(__ffsll((long long)t) - 1);
        t &= t - 1ull;
        atomicAdd(&waves[w].lws_touched, 1u);
        if (!(d.z & kDenseEvaluated)) continue;
        const int32_t after = clamp_i32((int64_t)(int32_t)d.x - __ldcg(p.lost + (size_t)i * p.cols + w));
        atomicMin(&waves[w].min_margin, clamp_i32((int64_t)after - (int32_t)d.y));
        if ((d.z & kDenseAvailable) && ((nb >> w) & 1ull)) atomicAdd(&waves[w].lws_loses_available, 1u);
      }
    }
    if (i < p.m) {
      const lwse_drain_wave_key* k = reinterpret_cast<const lwse_drain_wave_key*>(p.out + 16) + i;
      const uint32_t w = k->wave;
      if (w == LWSE_NONE) continue;
      const lwse_drain_budget_cost* c = p.cost + k->id;
      atomicAdd(&waves[w].n_pods_evicted, __ldg(&c->pods));
      atomicAdd(&waves[w].n_leaders_evicted, __ldg(&c->leaders));
    }
  }
}

__global__ void __launch_bounds__(256) drain_waves_fill_capped_kernel(const DrainWavesLaunch p, const uint32_t* caps) {
  drain_waves_fill<true>(p, caps);
}

__global__ void __launch_bounds__(256) drain_waves_dense_capped_kernel(const DrainWavesLaunch p, const uint32_t* caps,
                                                                       uint32_t constraints) {
  drain_waves_dense<true>(p, caps, constraints);
}

__global__ void __launch_bounds__(kPlanThreads, 1) drain_waves_plan_capped_kernel(const DrainWavesLaunch p) {
  drain_waves_plan<true>(p);
}

int launch_drain_waves_capped(const DrainWavesLaunch* p, const uint32_t* caps, uint32_t constraints, int pass, int sm_count,
                              cudaStream_t s) {
  if (pass == 1) {
    drain_waves_fill_capped_kernel<<<grid_for(p->n_pairs, 256, (uint32_t)sm_count * 8u), 256, 0, s>>>(*p, caps);
    if (const int r = launch_result(1); r < 0) return r;
    if (const int r = launch_index_scan(p->l_count, p->l_first, p->l_cursor, p->n_lws, s); r < 0) return r;
    const uint64_t n = p->n_lws > p->n_pairs ? p->n_lws : p->n_pairs;
    drain_waves_dense_capped_kernel<<<grid_for(n, 256, (uint32_t)sm_count * 8u), 256, 0, s>>>(*p, caps, constraints);
    return launch_result(3);
  }
  drain_waves_plan_capped_kernel<<<1, kPlanThreads, 0, s>>>(*p);
  const uint32_t n = p->n_dense > p->m ? p->n_dense : p->m;
  drain_waves_finish_kernel<<<grid_for(n, 256, (uint32_t)sm_count * 4u), 256, 0, s>>>(*p);
  return launch_result(2);
}

int launch_drain_waves_finish(const DrainWavesLaunch* p, int sm_count, cudaStream_t s) {
  const uint32_t n = p->n_dense > p->m ? p->n_dense : p->m;
  drain_waves_finish_kernel<<<grid_for(n, 256, (uint32_t)sm_count * 4u), 256, 0, s>>>(*p);
  return launch_result(1);
}

int launch_drain_waves(const DrainWavesLaunch* p, int pass, int sm_count, cudaStream_t s) {
  switch (pass) {
    case 0: {
      const uint32_t n = p->m > p->n_keys ? p->m : p->n_keys;
      drain_waves_keys_kernel<<<grid_for(n, 256, (uint32_t)sm_count * 4u), 256, 0, s>>>(*p);
      if (const int r = launch_result(1); r < 0) return r;
      if (const int r = launch_index_scan(p->count, p->first, p->cursor, p->m, s); r < 0) return r;
      return 2;
    }
    case 1: {
      drain_waves_fill_kernel<<<grid_for(p->n_pairs, 256, (uint32_t)sm_count * 8u), 256, 0, s>>>(*p);
      if (const int r = launch_result(1); r < 0) return r;
      if (const int r = launch_index_scan(p->l_count, p->l_first, p->l_cursor, p->n_lws, s); r < 0) return r;
      const uint64_t n = p->n_lws > p->n_pairs ? p->n_lws : p->n_pairs;
      drain_waves_dense_kernel<<<grid_for(n, 256, (uint32_t)sm_count * 8u), 256, 0, s>>>(*p);
      return launch_result(3);
    }
    default: {
      drain_waves_plan_kernel<<<1, kPlanThreads, 0, s>>>(*p);
      const uint32_t n = p->n_dense > p->m ? p->n_dense : p->m;
      drain_waves_finish_kernel<<<grid_for(n, 256, (uint32_t)sm_count * 4u), 256, 0, s>>>(*p);
      return launch_result(2);
    }
  }
}

}  // namespace lwse
