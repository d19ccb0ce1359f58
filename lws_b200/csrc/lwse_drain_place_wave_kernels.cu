// Drain placement waves (lwse_resident_drain_place_waves, sm_90a); the definition is in lwse.h, the argument in
// DESIGN.md §3.5, "Drain placement waves".
//
// Setup (after the drain waves chain up to its dense rows and the drain placement's passes, which give the alone
// rows of every key):
//   dpw_domain_count_kernel / dpw_domain_fill_kernel   the rule-(b) rows (not pinned, PLACED in the baseline, of a
//                              namespace) indexed by their baseline domain (count, scan, fill).
//   dpw_init_kernel            the column rows of the first step.
// One step per key, captured once as a graph and replayed with the key cursor in device memory:
//   dpw_floor_kernel           one CTA: the drain waves plan's add and check passes for this key over one column per
//                              open wave and one for the key alone.
//   dpw_items_kernel           per column, the namespaces of W_c ∪ {k} by (a) / (b) from the wave state and k's own
//                              contribution (items only for open waves whose floor the constraints keep; the flags
//                              of the key-alone column too, for a wave the key may open).
//   place_ns_kernel<false, true, true, true>   the set-overlay solve of the items into the column rows.
//   dpw_commit_kernel          one CTA: the first feasible column, the plan body's commit of the floor state, U_k,
//                              N_k, the drained free slots and the namespaces into the wave, the column's placement
//                              counts into the wave row; the column state cleared for the next key.
// Finish: the drain waves finish, the wave rows' lws_breached, and the answer assembled.
#include "lwse_device.cuh"
#include "lwse_launch.cuh"

namespace lwse {

// (the pair record bits and dense flags of lwse_drain_wave_kernels.cu)
constexpr uint32_t kPairMember = 1u << 0;
constexpr uint32_t kPairReady = 1u << 1;
constexpr uint32_t kPairReadyNb = 1u << 2;
constexpr uint32_t kPairBound = 1u << 3;
constexpr uint32_t kStepThreads = 512;

__device__ __forceinline__ uint32_t dpw_node_free(const DrainPlaceLaunch& p, uint32_t n) {
  const uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(p.nodes + n) + 3);  // capacity | flags << 16
  const uint32_t cap = w & 0xFFFFu, occ = p.occupancy ? __ldg(p.occupancy + n) : 0u;
  return cap > occ ? cap - occ : 0u;
}

// A rule-(b) row: not pinned, of a namespace, PLACED in a domain of the baseline.  Its domain, or LWSE_NONE.
__device__ __forceinline__ uint32_t dpw_b_domain(const DrainPlaceLaunch& p, uint32_t r) {
  const uint4 hi = __ldg(reinterpret_cast<const uint4*>(p.reqs + r) + 1);
  if (hi.w != LWSE_NONE || hi.y >= p.n_namespaces) return LWSE_NONE;
  const uint4 o = __ldg(reinterpret_cast<const uint4*>(p.base + r));
  return ((o.z & LWSE_PLACE_PLACED) && o.x < p.n_domains) ? o.x : LWSE_NONE;
}

__global__ void __launch_bounds__(256) dpw_domain_count_kernel(const DrainPlaceWavesLaunch d) {
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < d.p.n_reqs; r += gridDim.x * blockDim.x) {
    const uint32_t dom = dpw_b_domain(d.p, r);
    if (dom != LWSE_NONE) atomicAdd(d.dix_count + dom, 1u);
  }
}

__global__ void __launch_bounds__(256) dpw_domain_fill_kernel(const DrainPlaceWavesLaunch d) {
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < d.p.n_reqs; r += gridDim.x * blockDim.x) {
    const uint32_t dom = dpw_b_domain(d.p, r);
    if (dom != LWSE_NONE) d.dix_rows[atomicAdd(d.dix_cursor + dom, 1u)] = r;
  }
}

// Column c's row at the start of a step: the wave's |U_W| and the counts of its rows of no namespace, with the
// baseline totals under PLACED / UNSCHEDULABLE / CONFLICT (the solve adds deltas).
__device__ __forceinline__ void dpw_reset_columns(const DrainPlaceWavesLaunch& d, uint32_t tid) {
  for (uint32_t j = tid; j < LWSE_DRAIN_WAVES_MAX * 16u; j += blockDim.x) {
    const uint32_t f = j & 15u;
    uint32_t v = (f >= 1u && f <= 10u) ? d.wnons[j] : 0u;
    if (f >= 8u && f <= 10u) v += __ldcg(d.p.counts + (f - 8u));
    d.col_rows[j] = v;
  }
}

__global__ void __launch_bounds__(256) dpw_init_kernel(const DrainPlaceWavesLaunch d) { dpw_reset_columns(d, threadIdx.x); }

// 1. The floor columns: the drain waves plan's passes 1 and 2 for key position i (drain_waves_plan).
__global__ void __launch_bounds__(kStepThreads, 1) dpw_floor_kernel(const DrainPlaceWavesLaunch d) {
  const DrainWavesLaunch& p = d.w;
  DpwState* st = d.st;
  const uint32_t tid = threadIdx.x, i = st->i, n_open = st->n_open;
  if (i >= p.m) return;
  if (tid == 0) st->key = __ldg(p.ids + i);
  const uint32_t b = __ldg(p.first + i), e = __ldg(p.first + i + 1);
  const uint32_t cols = n_open + 1, items = (e - b) * cols;
  for (uint32_t j = tid; j < items; j += kStepThreads) {
    const uint4 r = __ldg(p.recs + b + j / cols);
    const uint32_t w = j % cols;
    if (w == 0 && (r.z & kPairMember) && atomicExch(p.stamps + 2u * r.y, i + 1u) != i + 1u) atomicAdd(&st->touched, 1u);
    if ((r.z & kPairBound) && (w == n_open || !((__ldcg(p.g_waves + r.x) >> w) & 1ull)))
      atomicAdd(p.lost + (size_t)r.y * p.cols + w, 1u);
  }
  __syncthreads();
  for (uint32_t j = tid; j < items; j += kStepThreads) {
    const uint4 r = __ldg(p.recs + b + j / cols);
    const uint32_t w = j % cols;
    if (!(r.z & kPairBound) || !(w == n_open || !((__ldcg(p.g_waves + r.x) >> w) & 1ull))) continue;
    const uint4 dr = __ldg(p.dense + r.y);
    if ((int64_t)__ldcg(p.lost + (size_t)r.y * p.cols + w) <= (int64_t)(int32_t)dr.x - (int32_t)dr.y) continue;
    if (w < n_open) {
      atomicOr(&st->bad, 1ull << w);
    } else {
      st->alone_bad = 1u;
      if (atomicExch(p.stamps + 2u * r.y + 1u, i + 1u) != i + 1u) atomicAdd(&st->breached, 1u);
    }
  }
}

__device__ __forceinline__ void dpw_item(const DrainPlaceWavesLaunch& d, uint32_t c, uint32_t ns, bool emit) {
  if (atomicExch(d.col_ns + (size_t)c * d.p.n_namespaces + ns, 1u) != 0u || !emit) return;
  const uint32_t at = atomicAdd(&d.st->n_items, 1u);
  if (at < d.item_capacity) d.items[at] = make_uint2(c, ns);
  else atomicAdd(&d.st->refused, 1u);
}

// 2. The items.  Column c < n_open is wave c with k added (solved when its floor is kept or not constrained);
// column n_open, when a new wave may open, is {k} alone: only its namespace flags are set (its counts are the
// key's alone row).  Every bit and slot of a wave that is not open is zero, so one rule serves both.
__global__ void __launch_bounds__(256) dpw_items_kernel(const DrainPlaceWavesLaunch d) {
  const DrainPlaceLaunch& p = d.p;
  const DpwState* st = d.st;
  const uint32_t i = st->i;
  if (i >= d.w.m) return;
  const uint32_t k = st->key, n_open = st->n_open;
  const uint32_t cols = n_open < d.max_waves ? n_open + 1u : n_open;
  const unsigned long long bad = (d.constraints & LWSE_DPW_LWS_FLOOR) ? st->bad : 0ull;
  const uint32_t uf = __ldg(p.u_first + k), nu = __ldg(p.u_first + k + 1u) - uf;
  // k's domain (the only one whose rule-(b) rows k can add), and k's usable free slots
  uint32_t kd = LWSE_NONE, kf = 0;
  if (p.by_domain) {
    kd = k;
  } else {
    const uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(p.nodes + k) + 3), dom = __ldg(&p.nodes[k].domain_id);
    kd = dom < p.n_domains ? dom : LWSE_NONE;
    if (kd != LWSE_NONE && ((w >> 16) & LWSE_NODE_SCHEDULABLE) && ((w >> 16) & LWSE_NODE_HAS_TOPOLOGY)) kf = dpw_node_free(p, k);
  }
  const uint32_t bf = kd != LWSE_NONE ? __ldg(d.dix_first + kd) : 0u, nb = kd != LWSE_NONE ? __ldg(d.dix_first + kd + 1u) - bf : 0u;
  const uint32_t per = p.n_namespaces + nu + nb;
  const uint64_t total = (uint64_t)per * cols;
  for (uint64_t j = blockIdx.x * blockDim.x + threadIdx.x; j < total; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t c = (uint32_t)(j / per), x = (uint32_t)(j % per);
    const bool emit = c < n_open;
    if (emit && ((bad >> c) & 1ull)) continue;
    const unsigned long long bit = 1ull << c;
    if (x < p.n_namespaces) {  // (a) and (b) of W_c: the wave's namespaces
      if (__ldcg(d.ns_wave + x) & bit) dpw_item(d, c, x, emit);
    } else if (x < p.n_namespaces + nu) {  // (a) of k: U_k
      const uint32_t r = __ldg(p.u_rows + uf + (x - p.n_namespaces));
      const uint32_t ns = __ldg(&p.reqs[r].ns);
      if (ns < p.n_namespaces) {
        dpw_item(d, c, ns, emit);
      } else if (emit && !(__ldcg(d.u_wave + r) & bit)) {  // no namespace: UNSCHEDULABLE without a solve
        uint32_t cnt[kDrainCounts] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
        drain_place_count(cnt, __ldg(reinterpret_cast<const uint4*>(p.base + r)),
                          make_uint4(LWSE_NONE, LWSE_NONE, LWSE_PLACE_UNSCHEDULABLE, 0u), true);
        for (uint32_t f = 0; f < kDrainCounts; f++)
          if (cnt[f]) atomicAdd(d.col_rows + c * 16u + 2u + f, cnt[f]);
      }
      if (emit && !(__ldcg(d.u_wave + r) & bit)) atomicAdd(d.col_rows + c * 16u + 1u, 1u);
    } else {  // (b) of k: the rows PLACED in k's domain
      const uint32_t r = __ldg(d.dix_rows + bf + (x - p.n_namespaces - nu));
      bool hit = p.by_domain;
      if (!hit) {
        const uint32_t m = __ldg(&p.base[r].leader_node);
        const uint32_t drained = __ldcg(d.drained + (size_t)c * p.n_domains + kd) + kf;
        hit = m == k || (m < p.n_nodes && (__ldcg(d.key_wave + m) & bit)) ||
              (int64_t)__ldcg(p.dom_free + kd) - (int64_t)drained < (int64_t)(int32_t)__ldg(&p.reqs[r].size);
      }
      if (hit) dpw_item(d, c, __ldg(&p.reqs[r].ns), emit);
    }
  }
}

// 4. Choose and commit, then clear the column state for the next key.
__global__ void __launch_bounds__(kStepThreads, 1) dpw_commit_kernel(const DrainPlaceWavesLaunch d) {
  const DrainWavesLaunch& p = d.w;
  const DrainPlaceLaunch& pp = d.p;
  DpwState* st = d.st;
  __shared__ uint32_t s_wave, s_new;
  const uint32_t tid = threadIdx.x, i = st->i, n_open = st->n_open;
  if (i >= p.m) return;
  const uint32_t k = st->key;
  const uint32_t* alone_row = reinterpret_cast<const uint32_t*>(pp.rows + k);
  if (tid == 0) {
    uint32_t alone = st->alone_bad ? LWSE_DPW_LWS_FLOOR : 0u;
    if (__ldcg(alone_row + 2)) alone |= LWSE_DPW_STRANDED;
    if (__ldcg(alone_row + 3)) alone |= LWSE_DPW_BUMPED;
    uint32_t wave = LWSE_NONE, status = LWSE_DRAINW_BREACHES_ALONE;
    if (!(alone & d.constraints)) {
      status = LWSE_DRAINW_PLANNED;
      for (uint32_t c = 0; c < n_open && wave == LWSE_NONE; c++) {
        const uint32_t* col = d.col_rows + c * 16u;
        if ((d.constraints & LWSE_DPW_LWS_FLOOR) && ((st->bad >> c) & 1ull)) continue;
        if ((d.constraints & LWSE_DPW_STRANDED) && col[2]) continue;
        if ((d.constraints & LWSE_DPW_BUMPED) && col[3]) continue;
        wave = c;
      }
      if (wave == LWSE_NONE) {
        if (n_open < d.max_waves) wave = n_open;
        else status = LWSE_DRAINW_NO_WAVE;
      }
    }
    s_wave = wave;
    s_new = wave == n_open ? 1u : 0u;
    d.kalone[i] = alone;
    st->status[status]++;
    uint32_t* row = reinterpret_cast<uint32_t*>(p.out + 16 + (size_t)i * sizeof(lwse_drain_wave_key));
    row[1] = wave;
    row[2] = status;
    row[5] = st->touched;
    row[6] = st->breached;
    if (wave != LWSE_NONE) {
      uint32_t* wrow = reinterpret_cast<uint32_t*>(p.out + 16 + (size_t)p.m * sizeof(lwse_drain_wave_key) +
                                                   (size_t)wave * sizeof(lwse_drain_wave));
      wrow[0]++;
      if (s_new) wrow[7] = (uint32_t)INT32_MAX;
      const uint32_t* src = s_new ? alone_row : d.col_rows + wave * 16u;  // the committed probe's counts
      uint32_t* dst = d.wplace + wave * 16u;
      for (uint32_t f = 1; f < 12; f++) dst[f] = __ldcg(src + f);
    }
  }
  __syncthreads();
  const uint32_t wave = s_wave;
  // the plan body's pass 4: the other floor columns taken back; the key's groups join its wave
  const uint32_t b = __ldg(p.first + i), e = __ldg(p.first + i + 1);
  const uint32_t cols = n_open + 1, items = (e - b) * cols;
  uint8_t* wrows = p.out + 16 + (size_t)p.m * sizeof(lwse_drain_wave_key);
  for (uint32_t j = tid; j < items; j += kStepThreads) {
    const uint4 r = __ldg(p.recs + b + j / cols);
    const uint32_t w = j % cols;
    if (w != wave) {
      if ((r.z & kPairBound) && (w == n_open || !((__ldcg(p.g_waves + r.x) >> w) & 1ull)))
        atomicSub(p.lost + (size_t)r.y * p.cols + w, 1u);
      continue;
    }
    const unsigned long long bit = 1ull << w;
    if (!(atomicOr(p.g_waves + r.x, bit) & bit)) {
      lwse_drain_wave* wr = reinterpret_cast<lwse_drain_wave*>(wrows) + w;
      atomicAdd(&wr->n_groups_restarted, 1u);
      if (r.z & kPairReady) atomicAdd(&wr->n_ready_restarted, 1u);
      atomicAdd(reinterpret_cast<unsigned long long*>(&wr->n_pods_recreated), (unsigned long long)r.w);
    }
    if (r.z & kPairMember) {
      atomicOr(p.row_waves + 2u * r.y, bit);
      if (r.z & kPairReadyNb) atomicOr(p.row_waves + 2u * r.y + 1u, bit);
    }
  }
  if (wave != LWSE_NONE) {
    const unsigned long long bit = 1ull << wave;
    // U_k into the wave (its rows of no namespace keep their counts in wnons), N_k, the drained free slots
    for (uint32_t j = __ldg(pp.u_first + k) + tid, end = __ldg(pp.u_first + k + 1u); j < end; j += kStepThreads) {
      const uint32_t r = __ldg(pp.u_rows + j);
      if (atomicOr(d.u_wave + r, bit) & bit) continue;
      atomicAdd(d.wnons + wave * 16u + 1u, 1u);
      if (__ldg(&pp.reqs[r].ns) < pp.n_namespaces) continue;
      uint32_t cnt[kDrainCounts] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
      drain_place_count(cnt, __ldg(reinterpret_cast<const uint4*>(pp.base + r)),
                        make_uint4(LWSE_NONE, LWSE_NONE, LWSE_PLACE_UNSCHEDULABLE, 0u), true);
      for (uint32_t f = 0; f < kDrainCounts; f++)
        if (cnt[f]) atomicAdd(d.wnons + wave * 16u + 2u + f, cnt[f]);
    }
    if (tid == 0) {
      d.key_wave[k] |= bit;
      if (!pp.by_domain) {
        const uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(pp.nodes + k) + 3), dom = __ldg(&pp.nodes[k].domain_id);
        if (dom < pp.n_domains && ((w >> 16) & LWSE_NODE_SCHEDULABLE) && ((w >> 16) & LWSE_NODE_HAS_TOPOLOGY))
          d.drained[(size_t)wave * pp.n_domains + dom] += dpw_node_free(pp, k);
      }
    }
    for (uint32_t ns = tid; ns < pp.n_namespaces; ns += kStepThreads)
      if (__ldcg(d.col_ns + (size_t)wave * pp.n_namespaces + ns)) d.ns_wave[ns] |= bit;
  }
  __syncthreads();
  // the column state of this key cleared; the next key's columns start from the waves
  const uint32_t n_cols = n_open < d.max_waves ? n_open + 1u : n_open;
  for (uint32_t j = tid; j < n_cols * pp.n_namespaces; j += kStepThreads) d.col_ns[j] = 0u;
  dpw_reset_columns(d, tid);
  if (tid == 0) {
    st->i = i + 1u;
    if (s_new) st->n_open = n_open + 1u;
    st->n_items = 0u;
    st->bad = 0ull;
    st->alone_bad = st->touched = st->breached = 0u;
  }
}

// lws_breached per wave: the evaluated dense rows whose lost groups pass their slack.
__global__ void __launch_bounds__(256) dpw_breached_kernel(const DrainPlaceWavesLaunch d) {
  const DrainWavesLaunch& p = d.w;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < p.n_dense; i += gridDim.x * blockDim.x) {
    const uint4 dr = __ldg(p.dense + i);
    if (!(dr.z & 1u)) continue;  // kDenseEvaluated
    unsigned long long t = p.row_waves[2u * i];
    while (t) {
      const uint32_t w = (uint32_t)(__ffsll((long long)t) - 1);
      t &= t - 1ull;
      if ((int64_t)__ldcg(p.lost + (size_t)i * p.cols + w) > (int64_t)(int32_t)dr.x - (int32_t)dr.y) atomicAdd(d.wbreach + w, 1u);
    }
  }
}

// The answer: totals, 48-byte key rows, 96-byte wave rows.
__global__ void __launch_bounds__(256) dpw_finish_kernel(const DrainPlaceWavesLaunch d) {
  const DrainWavesLaunch& p = d.w;
  const uint32_t n_open = d.st->n_open;
  const uint8_t* wkeys = p.out + 16;
  const lwse_drain_wave* wwaves = reinterpret_cast<const lwse_drain_wave*>(p.out + 16 + (size_t)p.m * sizeof(lwse_drain_wave_key));
  lwse_drain_place_wave_key* keys = reinterpret_cast<lwse_drain_place_wave_key*>(d.out + 16);
  lwse_drain_place_wave* waves = reinterpret_cast<lwse_drain_place_wave*>(d.out + 16 + (size_t)p.m * sizeof(lwse_drain_place_wave_key));
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < p.m || i < n_open; i += gridDim.x * blockDim.x) {
    if (i < p.m) {
      const lwse_drain_wave_key* s = reinterpret_cast<const lwse_drain_wave_key*>(wkeys) + i;
      const lwse_drain_place_cost* a = d.p.rows + s->id;
      lwse_drain_place_wave_key o;
      o.id = s->id;
      o.wave = s->wave;
      o.status = s->status;
      o.alone = d.kalone[i];
      o.groups_restarted = s->groups_restarted;
      o.ready_restarted = s->ready_restarted;
      o.lws_touched = s->lws_touched;
      o.lws_breached = s->lws_breached;
      o.unpinned = a->unpinned;
      o.stranded = a->stranded;
      o.bumped = a->bumped;
      o.reserved = 0u;
      keys[i] = o;
    }
    if (i < n_open) {
      const lwse_drain_wave s = wwaves[i];
      const uint32_t* pl = d.wplace + i * 16u;
      lwse_drain_place_wave o;
      o.n_keys = s.n_keys;
      o.lws_touched = s.lws_touched;
      o.lws_loses_available = s.lws_loses_available;
      o.n_pods_evicted = s.n_pods_evicted;
      o.n_leaders_evicted = s.n_leaders_evicted;
      o.n_groups_restarted = s.n_groups_restarted;
      o.n_ready_restarted = s.n_ready_restarted;
      o.min_margin = s.min_margin;
      o.n_pods_recreated = s.n_pods_recreated;
      o.lws_breached = d.wbreach[i];
      o.unpinned = pl[1];
      o.stranded = pl[2];
      o.bumped = pl[3];
      o.n_changed = pl[4];
      o.n_lost = pl[5];
      o.n_moved = pl[6];
      o.n_gained = pl[7];
      o.n_placed = pl[8];
      o.n_unschedulable = pl[9];
      o.n_conflict = pl[10];
      o.namespaces_solved = pl[11];
      o.reserved[0] = o.reserved[1] = 0u;
      waves[i] = o;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0)
    *reinterpret_cast<uint4*>(d.out) = make_uint4(n_open, d.st->status[LWSE_DRAINW_PLANNED], d.st->status[LWSE_DRAINW_BREACHES_ALONE],
                                                  d.st->status[LWSE_DRAINW_NO_WAVE]);
}

int launch_drain_place_waves(const DrainPlaceWavesLaunch* d, int pass, int sm_count, cudaStream_t s) {
  switch (pass) {
    case 0: {  // the rule-(b) domain index and the first step's columns
      const unsigned g = grid_for(d->p.n_reqs, 256, (uint32_t)sm_count * 8u);
      dpw_domain_count_kernel<<<g, 256, 0, s>>>(*d);
      if (const int r = launch_result(1); r < 0) return r;
      if (const int r = launch_index_scan(d->dix_count, d->dix_first, d->dix_cursor, d->p.n_domains, s); r < 0) return r;
      dpw_domain_fill_kernel<<<g, 256, 0, s>>>(*d);
      dpw_init_kernel<<<1, 256, 0, s>>>(*d);
      return launch_result(4);
    }
    case 1: {  // one step (captured into the step graph)
      dpw_floor_kernel<<<1, kStepThreads, 0, s>>>(*d);
      dpw_items_kernel<<<(unsigned)sm_count * 2u, 256, 0, s>>>(*d);
      if (const int r = launch_result(2); r < 0) return r;
      const int solved = launch_place_ns_drain_set(d, sm_count, s);
      if (solved < 0) return solved;
      dpw_commit_kernel<<<1, kStepThreads, 0, s>>>(*d);
      return launch_result(3 + solved);
    }
    default: {  // the finish
      if (const int r = launch_drain_waves_finish(&d->w, sm_count, s); r < 0) return r;
      dpw_breached_kernel<<<grid_for(d->w.n_dense, 256, (uint32_t)sm_count * 4u), 256, 0, s>>>(*d);
      const uint32_t n = d->w.m > LWSE_DRAIN_WAVES_MAX ? d->w.m : LWSE_DRAIN_WAVES_MAX;
      dpw_finish_kernel<<<grid_for(n, 256, (uint32_t)sm_count * 4u), 256, 0, s>>>(*d);
      return launch_result(3);
    }
  }
}

}  // namespace lwse
