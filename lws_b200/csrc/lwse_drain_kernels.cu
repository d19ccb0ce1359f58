// Drain what-if and drain cost (lwse_resident_drain_*, sm_90a); the definitions are in lwse.h.
//
//   drain_mark_kernel   the what-if's two changes, on its copies of the state column and the group rows:
//                       one pass over the identity rows (DELETING on pods bound to a marked node) and one
//                       over the group rows (POD_DELETING where the leader's node is marked).  The sweep
//                       (launch_lws_sweep) then runs over those copies.
//   drain_diff_kernel   the sweep's group rows against the baseline: changed rows appended with one atomic
//                       per warp, the restart counts reduced per warp before one atomic each.
//   drain_cost_kernel   every node at once, one warp per group: the group-level gate of handleRestartPolicy,
//                       then the group's pods 32 at a time (128-bit identity loads), the per-pod verdict of
//                       the group pass (lwse_restart.cuh) with the deleting bit set, and the group's
//                       restart nodes deduplicated (__match_any_sync per batch, a per-warp list across
//                       batches) before one atomic per (group, node) pair and field.
//
// Drain budget (lwse_resident_drain_budget*):
//   drain_domain_mask_kernel   the node mask of a set of domains, from the node rows' domain_id.
//   drain_budget_kernel        the set form, after the what-if's mark → sweep → diff: one warp per LWS row over
//                              its group range, the what-if rows against the baseline; touched rows appended
//                              with one atomic per LWS, the totals reduced per warp before one atomic each.
//   drain_budget_walk_kernel   the per-key form: drain_cost_kernel's walk (same gate, visit_pod, dedup) with
//                              the key = the node or its domain.  <false> adds the cost totals per key and
//                              counts the pairs; <true> adds every fresh (group, key) pair of a group that
//                              belongs to its LWS row into an open-addressing (LWS, key) table.
//   drain_budget_keys_init_kernel / drain_budget_finish_kernel   the key rows' pods and min_margin start; each
//                              table entry turned into its key's lws_touched / breached / loses / min_margin.
#include "lwse_device.cuh"
#include "lwse_launch.cuh"
#include "lwse_restart.cuh"

namespace lwse {

constexpr uint32_t kRestartBits = LWSE_GOUT_DELETE_LEADER | LWSE_GOUT_LEADER_DELETING;

__device__ __forceinline__ unsigned long long warp_sum_u64(unsigned long long v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, off);
  return v;
}

// --------------------------------------------------------------------------
// drain what-if: mark, then diff
// --------------------------------------------------------------------------
struct DrainMarkArgs {
  const uint8_t* mask;  // n_nodes bytes, 1 = the node is in D
  const lwse_pod_ident* ident;
  uint8_t* state;            // the what-if's copy of the state column
  lwse_group_rec* groups;    // the what-if's copy of the group rows
  uint32_t* counts;          // [1] pods evicted, [2] leaders evicted
  uint64_t n_pods;
  uint32_t n_groups, n_nodes;
};

__global__ void __launch_bounds__(256) drain_mark_kernel(const DrainMarkArgs a) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  const uint64_t first = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t pods = 0, leaders = 0;
  for (uint64_t p = first; p < a.n_pods; p += stride) {
    const uint32_t place = __ldcs(&a.ident[p].place);
    const uint32_t node = place >> LWSE_PODID_NODE_SHIFT;
    if ((place & LWSE_PODID_SCHEDULED) && node < a.n_nodes && __ldg(a.mask + node)) {
      a.state[p] |= (uint8_t)LWSE_POD_DELETING;
      pods++;
    }
  }
  for (uint64_t g = first; g < a.n_groups; g += stride) {
    const uint32_t node = a.groups[g].leader_node;
    if (node < a.n_nodes && __ldg(a.mask + node)) {
      a.groups[g].flags |= LWSE_GRP_POD_DELETING;
      leaders++;
    }
  }
  pods = __reduce_add_sync(0xFFFFFFFFu, pods);
  leaders = __reduce_add_sync(0xFFFFFFFFu, leaders);
  if (lane == 0 && pods) atomicAdd(a.counts + 1, pods);
  if (lane == 0 && leaders) atomicAdd(a.counts + 2, leaders);
}

int launch_drain_mark(const uint8_t* d_mask, uint32_t n_nodes, const lwse_pod_ident* d_ident, uint8_t* d_state, uint64_t n_pods,
                      lwse_group_rec* d_groups, uint32_t n_groups, uint32_t* d_counts, int sm_count, cudaStream_t s) {
  const DrainMarkArgs a{d_mask, d_ident, d_state, d_groups, d_counts, n_pods, n_groups, n_nodes};
  const uint64_t items = n_pods > n_groups ? n_pods : n_groups;
  drain_mark_kernel<<<grid_for(items, 256, (uint32_t)sm_count * 16u), 256, 0, s>>>(a);
  return launch_result(1);
}

struct DrainDiffArgs {
  const lwse_group_out* before;  // the baseline
  const lwse_group_out* after;   // the what-if's sweep
  const lwse_group_rec* groups;  // pod_count of the restarted groups
  uint32_t* rows;
  lwse_group_out* outs_before;
  lwse_group_out* outs_after;
  uint32_t* counts;  // [0] changed rows, [3] restarted, [4] ready restarted, [6..7] pods recreated (u64)
  uint32_t capacity, n_groups;
};

__global__ void __launch_bounds__(256) drain_diff_kernel(const DrainDiffArgs a) {
  const uint32_t lane = threadIdx.x & 31u, stride = gridDim.x * blockDim.x;
  uint32_t restarted = 0, ready = 0;
  unsigned long long pods = 0;
  for (uint32_t base = (blockIdx.x * blockDim.x + threadIdx.x) & ~31u; base < a.n_groups; base += stride) {
    const uint32_t r = base + lane;
    bool changed = false;
    uint4 v = make_uint4(0u, 0u, 0u, 0u), o = v;
    if (r < a.n_groups) {
      v = __ldcg(reinterpret_cast<const uint4*>(a.after + r));
      o = __ldcg(reinterpret_cast<const uint4*>(a.before + r));
      changed = v.x != o.x || v.y != o.y || v.z != o.z || v.w != o.w;
      if (!(o.x & kRestartBits) && (v.x & kRestartBits)) {
        restarted++;
        ready += (o.x & LWSE_GOUT_COND_READY) ? 1u : 0u;
        pods += __ldg(&a.groups[r].pod_count);
      }
    }
    const uint32_t mask = __ballot_sync(0xFFFFFFFFu, changed);
    if (mask == 0u) continue;  // warp-uniform
    uint32_t at = 0;
    if (lane == 0) at = atomicAdd(a.counts, (uint32_t)__popc(mask));
    at = __shfl_sync(0xFFFFFFFFu, at, 0) + (uint32_t)__popc(mask & ((1u << lane) - 1u));
    if (changed && at < a.capacity) {
      a.rows[at] = r;
      *reinterpret_cast<uint4*>(a.outs_before + at) = o;
      *reinterpret_cast<uint4*>(a.outs_after + at) = v;
    }
  }
  restarted = __reduce_add_sync(0xFFFFFFFFu, restarted);
  ready = __reduce_add_sync(0xFFFFFFFFu, ready);
  pods = warp_sum_u64(pods);
  if (lane == 0 && restarted) atomicAdd(a.counts + 3, restarted);
  if (lane == 0 && ready) atomicAdd(a.counts + 4, ready);
  if (lane == 0 && pods) atomicAdd(reinterpret_cast<unsigned long long*>(a.counts + 6), pods);
}

int launch_drain_diff(const lwse_group_out* d_before, const lwse_group_out* d_after, const lwse_group_rec* d_groups,
                      uint32_t n_groups, uint32_t* d_rows, lwse_group_out* d_outs_before, lwse_group_out* d_outs_after,
                      uint32_t capacity, uint32_t* d_counts, int sm_count, cudaStream_t s) {
  const DrainDiffArgs a{d_before, d_after, d_groups, d_rows, d_outs_before, d_outs_after, d_counts, capacity, n_groups};
  drain_diff_kernel<<<grid_for(n_groups, 256, (uint32_t)sm_count * 4u), 256, 0, s>>>(a);
  return launch_result(1);
}

// --------------------------------------------------------------------------
// drain cost of every node
// --------------------------------------------------------------------------
struct DrainCostArgs {
  const lwse_lws_rec* lws;
  const lwse_group_rec* groups;
  const uint8_t* pod_state;
  const lwse_pod_ident* pod_ident;
  const lwse_group_out* baseline;
  lwse_drain_cost* cost;  // n_nodes rows: pods filled in, every other field zero
  uint64_t n_pods;
  uint32_t n_lws, n_groups, n_nodes;
};

constexpr uint32_t kCostThreads = 256;
constexpr uint32_t kCostList = 64;  // distinct restart nodes one warp remembers per group

// The node row that draining would make pod p restart its group through, or LWSE_NONE: p is
// scheduled on a node of the table and the group pass's verdict on it, deleting, recreates the group.
__device__ __forceinline__ uint32_t restart_node(const DrainCostArgs& a, const VisitCtx& ctx, uint32_t p, bool valid) {
  if (!valid) return LWSE_NONE;
  const uint4 id = ldg_stream(a.pod_ident + p);
  const uint32_t node = id.w >> LWSE_PODID_NODE_SHIFT;  // < 2^22: never LWSE_NONE
  if (!(id.w & LWSE_PODID_SCHEDULED) || node >= a.n_nodes) return LWSE_NONE;
  bool cand;
  (void)visit_pod(ctx, (uint32_t)__ldg(a.pod_state + p) | LWSE_POD_DELETING, id, cand);
  return cand ? node : LWSE_NONE;
}

__global__ void __launch_bounds__(kCostThreads) drain_cost_kernel(const DrainCostArgs a) {
  __shared__ uint32_t s_list[kCostThreads / 32][kCostList];
  constexpr uint32_t kFull = 0xFFFFFFFFu;
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint32_t lt = (1u << lane) - 1u;
  uint32_t* list = s_list[warp];
  const uint32_t n_warps = gridDim.x * (kCostThreads / 32);
  for (uint32_t g = blockIdx.x * (kCostThreads / 32) + warp; g < a.n_groups; g += n_warps) {
    const uint4* row = reinterpret_cast<const uint4*>(a.groups + g);
    const uint4 ca = ldg_stream(row + 0), cb = ldg_stream(row + 1), cc = ldg_stream(row + 2), cd = ldg_stream(row + 3);
    const uint32_t leader_node = cc.y, pod_base = cc.z, pod_count = cc.w, lws_index = cd.x;
    if (lane == 0 && leader_node < a.n_nodes) atomicAdd(&a.cost[leader_node].leaders, 1u);
    if (lws_index >= a.n_lws || (uint64_t)pod_base + pod_count > a.n_pods || pod_count == 0) continue;  // BAD_TABLE / no pods
    const uint32_t before = __ldcs(&a.baseline[g].flags);
    if (before & kRestartBits) continue;  // restarting already: draining changes no count
    const uint4 L = ldg_cached(a.lws + lws_index);
    const uint32_t lflags = L.w;
    if (!restart_policy_on(lflags)) continue;
    // pendingPodsInGroup (:338-362), read only when it can close the gate
    bool pending = (uint32_t)(int32_t)L.z != pod_count;
    if (!pending && restart_suppressed(true, lflags)) {
      for (uint32_t i0 = 0; i0 < pod_count && !pending; i0 += 32) {
        const uint32_t st = i0 + lane < pod_count ? (uint32_t)__ldg(a.pod_state + pod_base + i0 + lane) : 0u;
        pending = __any_sync(kFull, (st & LWSE_POD_PHASE_MASK) == LWSE_POD_PHASE_PENDING);
      }
    }
    if (restart_suppressed(pending, lflags)) continue;
    VisitCtx ctx;
    visit_ctx_of(ctx, ca, cb, cc, cd);
    const bool ready = (before & LWSE_GOUT_COND_READY) != 0u;
    uint32_t n_list = 0;
    bool listed = true;  // the list holds every restart node of the batches so far
    for (uint32_t b0 = 0; b0 < pod_count; b0 += 32) {
      const uint32_t key = restart_node(a, ctx, pod_base + b0 + lane, b0 + lane < pod_count);
      const uint32_t peers = __match_any_sync(kFull, key);
      bool fresh = key != LWSE_NONE && lane == (uint32_t)(__ffs(peers) - 1);
      if (listed) {
        for (uint32_t j = 0; j < n_list; j++) fresh &= list[j] != key;
        const uint32_t add = __ballot_sync(kFull, fresh);
        if (n_list + (uint32_t)__popc(add) <= kCostList) {
          __syncwarp();
          if (fresh) list[n_list + (uint32_t)__popc(add & lt)] = key;
          __syncwarp();
          n_list += (uint32_t)__popc(add);
        } else {
          listed = false;  // warp-uniform; from here on the earlier batches are read again
        }
      }
      if (!listed) {
        for (uint32_t e0 = 0; e0 < b0; e0 += 32) {
          const uint32_t k2 = restart_node(a, ctx, pod_base + e0 + lane, true);
          for (int j = 0; j < 32; j++) fresh &= __shfl_sync(kFull, k2, j) != key;
        }
      }
      if (fresh) {
        lwse_drain_cost* c = a.cost + key;
        atomicAdd(&c->groups_restarted, 1u);
        if (ready) atomicAdd(&c->ready_restarted, 1u);
        atomicAdd(reinterpret_cast<unsigned long long*>(&c->pods_recreated), (unsigned long long)pod_count);
      }
    }
  }
}

int launch_drain_cost(const lwse_lws_rec* d_lws, uint32_t n_lws, const lwse_group_rec* d_groups, uint32_t n_groups,
                      const uint8_t* d_state, const lwse_pod_ident* d_ident, uint64_t n_pods, const lwse_group_out* d_baseline,
                      lwse_drain_cost* d_cost, uint32_t n_nodes, int sm_count, cudaStream_t s) {
  if (n_groups == 0) return 0;
  const DrainCostArgs a{d_lws, d_groups, d_state, d_ident, d_baseline, d_cost, n_pods, n_lws, n_groups, n_nodes};
  drain_cost_kernel<<<grid_for(n_groups, kCostThreads / 32, (uint32_t)sm_count * 8u), kCostThreads, 0, s>>>(a);
  return launch_result(1);
}

// --------------------------------------------------------------------------
// drain budget (lwse_resident_drain_budget*): the definitions are in lwse.h
// --------------------------------------------------------------------------
// The drain mask of a set of domains: node n is drained iff its domain_id is a marked id below n_domains.
struct DrainDomainMaskArgs {
  const uint8_t* domains;  // n_domains bytes, 1 = the domain is drained
  const lwse_node_rec* nodes;
  uint8_t* mask;           // n_nodes bytes
  uint32_t n_nodes, n_domains;
};

__global__ void __launch_bounds__(256) drain_domain_mask_kernel(const DrainDomainMaskArgs a) {
  for (uint32_t n = blockIdx.x * blockDim.x + threadIdx.x; n < a.n_nodes; n += gridDim.x * blockDim.x) {
    const uint32_t d = __ldg(&a.nodes[n].domain_id);
    a.mask[n] = (d < a.n_domains && __ldg(a.domains + d)) ? 1u : 0u;
  }
}

int launch_drain_domain_mask(const uint8_t* d_domains, uint32_t n_domains, const lwse_node_rec* d_nodes, uint32_t n_nodes,
                             uint8_t* d_mask, int sm_count, cudaStream_t s) {
  const DrainDomainMaskArgs a{d_domains, d_nodes, d_mask, n_nodes, n_domains};
  drain_domain_mask_kernel<<<grid_for(n_nodes, 256, (uint32_t)sm_count * 4u), 256, 0, s>>>(a);
  return launch_result(1);
}

// The set form: one warp per LWS row over its group range, the what-if rows against the baseline.
struct DrainBudgetArgs {
  const lwse_lws_rec* lws;
  const lwse_lws_out* lws_out;   // the baseline
  const lwse_group_rec* groups;  // lws_index of every row
  const lwse_group_out* before;  // the baseline
  const lwse_group_out* after;   // the what-if's sweep
  lwse_drain_budget* rows;
  uint32_t* counts;  // [8] touched (the append cursor) [9] breached [10] loses available [11] already below
  uint32_t capacity, n_lws, n_groups;
};

__global__ void __launch_bounds__(256) drain_budget_kernel(const DrainBudgetArgs a) {
  constexpr uint32_t kFull = 0xFFFFFFFFu;
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t n_warps = gridDim.x * (blockDim.x / 32);
  uint32_t breached = 0, loses = 0, below = 0;  // lane 0's
  for (uint32_t L = (blockIdx.x * blockDim.x + threadIdx.x) / 32; L < a.n_lws; L += n_warps) {
    const LwsBudget b = budget_of(a.lws, a.lws_out, L, a.n_groups);
    uint32_t restarted = 0, lost = 0, lost_nb = 0;
    for (uint32_t i = lane; i < b.gcount; i += 32) {
      const uint32_t g = b.gbase + i;
      if (__ldg(&a.groups[g].lws_index) != L) continue;
      const uint32_t o = __ldcg(&a.before[g].flags), v = __ldcg(&a.after[g].flags);
      if (!(o & kRestartBits) && (v & kRestartBits)) {
        restarted++;
        if (o & LWSE_GOUT_COND_READY) {
          lost++;
          if ((int64_t)i < b.replicas) lost_nb++;
        }
      }
    }
    restarted = __reduce_add_sync(kFull, restarted);
    lost = __reduce_add_sync(kFull, lost);
    lost_nb = __reduce_add_sync(kFull, lost_nb);
    if (lane != 0) continue;
    const int32_t after = clamp_i32((int64_t)b.ready_before - lost);
    uint32_t flags = 0;
    if (!b.evaluated) {
      flags = LWSE_DRAINB_NOT_EVALUATED;
    } else {
      if (b.ready_before < b.floor) flags |= LWSE_DRAINB_ALREADY_BELOW;
      if (lost > 0 && after < b.floor) flags |= LWSE_DRAINB_BREACHED;
      if (b.available && lost_nb > 0) flags |= LWSE_DRAINB_LOSES_AVAILABLE;
      below += (flags & LWSE_DRAINB_ALREADY_BELOW) ? 1u : 0u;
    }
    if (restarted == 0) continue;
    breached += (flags & LWSE_DRAINB_BREACHED) ? 1u : 0u;
    loses += (flags & LWSE_DRAINB_LOSES_AVAILABLE) ? 1u : 0u;
    const uint32_t at = atomicAdd(a.counts + 8, 1u);
    if (at < a.capacity) {
      uint4* out = reinterpret_cast<uint4*>(a.rows + at);
      out[0] = make_uint4(L, flags, (uint32_t)b.replicas, (uint32_t)b.floor);
      out[1] = make_uint4((uint32_t)b.ready_before, (uint32_t)after, restarted, 0u);
    }
  }
  if (lane == 0 && breached) atomicAdd(a.counts + 9, breached);
  if (lane == 0 && loses) atomicAdd(a.counts + 10, loses);
  if (lane == 0 && below) atomicAdd(a.counts + 11, below);
}

int launch_drain_budget(const lwse_lws_rec* d_lws, const lwse_lws_out* d_lws_out, uint32_t n_lws, const lwse_group_rec* d_groups,
                        const lwse_group_out* d_before, const lwse_group_out* d_after, uint32_t n_groups,
                        lwse_drain_budget* d_rows, uint32_t capacity, uint32_t* d_counts, int sm_count, cudaStream_t s) {
  if (n_lws == 0) return 0;
  const DrainBudgetArgs a{d_lws, d_lws_out, d_groups, d_before, d_after, d_rows, d_counts, capacity, n_lws, n_groups};
  drain_budget_kernel<<<grid_for(n_lws, 256 / 32, (uint32_t)sm_count * 8u), 256, 0, s>>>(a);
  return launch_result(1);
}

// The per-key form.  The walk is drain_cost_kernel's with the restart node mapped to its key (the node, or
// its domain); the first pass adds the cost totals and counts the (group, key) pairs of groups that belong
// to their LWS row, the second inserts those pairs into an (LWS, key) table, and the finish pass turns
// every table entry into its key's budget columns.
struct DrainBudgetCostArgs {
  const lwse_lws_rec* lws;
  const lwse_lws_out* lws_out;
  const lwse_group_rec* groups;
  const uint8_t* pod_state;
  const lwse_pod_ident* pod_ident;
  const lwse_group_out* baseline;
  const lwse_node_rec* nodes;    // scope DOMAINS: key = nodes[node].domain_id when < n_domains; null: key = node
  lwse_drain_budget_cost* cost;  // n_keys rows
  unsigned long long* keys;      // the table: LWS row << 32 | key, kEmptyKey when free
  uint4* vals;                   // {groups restarted, ready groups restarted, of those with index < replicas, 0}
  uint32_t* counts;              // [0..1] pairs (u64), [2] refused inserts; pair mode: [8] pairs written
  uint64_t n_pods;
  uint32_t n_lws, n_groups, n_nodes, n_domains, table_mask;  // pair mode: keys = the pair list, table_mask its capacity
};

constexpr unsigned long long kEmptyKey = ~0ull;

__device__ __forceinline__ uint32_t key_of_node(const DrainBudgetCostArgs& a, uint32_t node) {
  if (node >= a.n_nodes) return LWSE_NONE;
  if (!a.nodes) return node;
  const uint32_t d = __ldg(&a.nodes[node].domain_id);
  return d < a.n_domains ? d : LWSE_NONE;
}

__device__ __forceinline__ uint32_t restart_key(const DrainBudgetCostArgs& a, const VisitCtx& ctx, uint32_t p, bool valid) {
  if (!valid) return LWSE_NONE;
  const uint4 id = ldg_stream(a.pod_ident + p);
  const uint32_t node = id.w >> LWSE_PODID_NODE_SHIFT;
  if (!(id.w & LWSE_PODID_SCHEDULED) || node >= a.n_nodes) return LWSE_NONE;
  bool cand;
  (void)visit_pod(ctx, (uint32_t)__ldg(a.pod_state + p) | LWSE_POD_DELETING, id, cand);
  return cand ? key_of_node(a, node) : LWSE_NONE;
}

__device__ __forceinline__ uint32_t table_slot(unsigned long long k, uint32_t mask) {
  k ^= k >> 33;
  k *= 0xFF51AFD7ED558CCDull;
  k ^= k >> 33;
  return (uint32_t)k & mask;
}

__device__ __forceinline__ void table_add(const DrainBudgetCostArgs& a, unsigned long long k, uint32_t ready, uint32_t ready_nb) {
  uint32_t h = table_slot(k, a.table_mask);
  for (uint32_t probe = 0; probe <= a.table_mask; probe++, h = (h + 1u) & a.table_mask) {
    const unsigned long long prev = atomicCAS(a.keys + h, kEmptyKey, k);
    if (prev == kEmptyKey || prev == k) {
      atomicAdd(&a.vals[h].x, 1u);
      if (ready) atomicAdd(&a.vals[h].y, 1u);
      if (ready_nb) atomicAdd(&a.vals[h].z, 1u);
      return;
    }
  }
  atomicAdd(a.counts + 2, 1u);  // full: the call fails
}

// kPairs: every fresh (group, key) pair of every group, member or not, as key << 32 | group into keys[0 ..
// table_mask) (the drain placement's restarts; the struct stays as the other instances read it).
template <bool kInsert, bool kPairs = false>
__global__ void __launch_bounds__(kCostThreads) drain_budget_walk_kernel(const DrainBudgetCostArgs a) {
  __shared__ uint32_t s_list[kCostThreads / 32][kCostList];
  constexpr uint32_t kFull = 0xFFFFFFFFu;
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint32_t lt = (1u << lane) - 1u;
  uint32_t* list = s_list[warp];
  const uint32_t n_warps = gridDim.x * (kCostThreads / 32);
  unsigned long long pairs = 0;
  for (uint32_t g = blockIdx.x * (kCostThreads / 32) + warp; g < a.n_groups; g += n_warps) {
    const uint4* row = reinterpret_cast<const uint4*>(a.groups + g);
    const uint4 ca = ldg_stream(row + 0), cb = ldg_stream(row + 1), cc = ldg_stream(row + 2), cd = ldg_stream(row + 3);
    const uint32_t leader_node = cc.y, pod_base = cc.z, pod_count = cc.w, lws_index = cd.x;
    if (!kInsert && !kPairs && lane == 0) {
      const uint32_t lk = key_of_node(a, leader_node);
      if (lk != LWSE_NONE) atomicAdd(&a.cost[lk].leaders, 1u);
    }
    if (lws_index >= a.n_lws || (uint64_t)pod_base + pod_count > a.n_pods || pod_count == 0) continue;
    const uint32_t before = __ldcs(&a.baseline[g].flags);
    if (before & kRestartBits) continue;
    const uint4 L = ldg_cached(a.lws + lws_index);
    const uint32_t lflags = L.w;
    if (!restart_policy_on(lflags)) continue;
    bool pending = (uint32_t)(int32_t)L.z != pod_count;
    if (!pending && restart_suppressed(true, lflags)) {
      for (uint32_t i0 = 0; i0 < pod_count && !pending; i0 += 32) {
        const uint32_t st = i0 + lane < pod_count ? (uint32_t)__ldg(a.pod_state + pod_base + i0 + lane) : 0u;
        pending = __any_sync(kFull, (st & LWSE_POD_PHASE_MASK) == LWSE_POD_PHASE_PENDING);
      }
    }
    if (restart_suppressed(pending, lflags)) continue;
    // the group belongs to its LWS row when the row's range is inside the table and holds g
    const uint4* lrow = reinterpret_cast<const uint4*>(a.lws + lws_index);
    const uint4 l1 = ldg_cached(lrow + 1), l3 = ldg_cached(lrow + 3);
    const uint32_t index = g - l3.z;
    const bool member = (uint64_t)l3.z + l3.w <= a.n_groups && g >= l3.z && index < l3.w;
    if (kInsert && !member) continue;
    VisitCtx ctx;
    visit_ctx_of(ctx, ca, cb, cc, cd);
    const bool ready = (before & LWSE_GOUT_COND_READY) != 0u;
    const bool ready_nb = ready && (int64_t)index < (int64_t)(int32_t)l1.x;
    uint32_t n_list = 0;
    bool listed = true;
    for (uint32_t b0 = 0; b0 < pod_count; b0 += 32) {
      const uint32_t key = restart_key(a, ctx, pod_base + b0 + lane, b0 + lane < pod_count);
      const uint32_t peers = __match_any_sync(kFull, key);
      bool fresh = key != LWSE_NONE && lane == (uint32_t)(__ffs(peers) - 1);
      if (listed) {
        for (uint32_t j = 0; j < n_list; j++) fresh &= list[j] != key;
        const uint32_t add = __ballot_sync(kFull, fresh);
        if (n_list + (uint32_t)__popc(add) <= kCostList) {
          __syncwarp();
          if (fresh) list[n_list + (uint32_t)__popc(add & lt)] = key;
          __syncwarp();
          n_list += (uint32_t)__popc(add);
        } else {
          listed = false;
        }
      }
      if (!listed) {
        for (uint32_t e0 = 0; e0 < b0; e0 += 32) {
          const uint32_t k2 = restart_key(a, ctx, pod_base + e0 + lane, true);
          for (int j = 0; j < 32; j++) fresh &= __shfl_sync(kFull, k2, j) != key;
        }
      }
      if (!fresh) continue;
      if (kPairs) {
        const uint32_t at = atomicAdd(a.counts + 8, 1u);
        if (at < a.table_mask) a.keys[at] = (unsigned long long)key << 32 | g;
      } else if (kInsert) {
        table_add(a, (unsigned long long)lws_index << 32 | key, ready, ready_nb);
      } else {
        lwse_drain_budget_cost* c = a.cost + key;
        atomicAdd(&c->groups_restarted, 1u);
        if (ready) atomicAdd(&c->ready_restarted, 1u);
        atomicAdd(reinterpret_cast<unsigned long long*>(&c->pods_recreated), (unsigned long long)pod_count);
        pairs += member ? 1u : 0u;
      }
    }
  }
  if (!kInsert && !kPairs) {
    pairs = warp_sum_u64(pairs);
    if (lane == 0 && pairs) atomicAdd(reinterpret_cast<unsigned long long*>(a.counts), pairs);
  }
}

// Every key row starts as {pods of its nodes, zeros, min_margin = INT32_MAX}; `cost` is zeroed by the caller.
__global__ void __launch_bounds__(256) drain_budget_keys_init_kernel(const DrainBudgetCostArgs a, const uint32_t* occupancy,
                                                                     uint32_t n_keys) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_keys || i < a.n_nodes; i += stride) {
    if (i < n_keys) a.cost[i].min_margin = INT32_MAX;
    if (i < a.n_nodes) {
      const uint32_t k = key_of_node(a, i), pods = __ldg(occupancy + i);
      if (k != LWSE_NONE && pods) atomicAdd(&a.cost[k].pods, pods);
    }
  }
}

__global__ void __launch_bounds__(256) drain_budget_finish_kernel(const DrainBudgetCostArgs a) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t h = blockIdx.x * blockDim.x + threadIdx.x; h <= a.table_mask; h += stride) {
    const unsigned long long k = a.keys[h];
    if (k == kEmptyKey) continue;
    const uint32_t L = (uint32_t)(k >> 32), key = (uint32_t)k;
    const uint4 v = a.vals[h];
    lwse_drain_budget_cost* c = a.cost + key;
    atomicAdd(&c->lws_touched, 1u);
    const LwsBudget b = budget_of(a.lws, a.lws_out, L, a.n_groups);
    if (!b.evaluated) continue;
    const int64_t after = (int64_t)b.ready_before - v.y;
    if (v.y > 0 && after < b.floor) atomicAdd(&c->lws_breached, 1u);
    if (b.available && v.z > 0) atomicAdd(&c->lws_loses_available, 1u);
    atomicMin(&c->min_margin, clamp_i32((int64_t)clamp_i32(after) - b.floor));
  }
}

int launch_drain_budget_cost(const DrainBudgetCostLaunch* p, int pass, int sm_count, cudaStream_t s) {
  const DrainBudgetCostArgs a{p->lws, p->lws_out, p->groups, p->pod_state, p->pod_ident, p->baseline,
                              p->by_domain ? p->nodes : nullptr, p->cost, p->keys, p->vals, p->counts,
                              p->n_pods, p->n_lws, p->n_groups, p->n_nodes, p->n_domains, p->table_mask};
  const unsigned walk_grid = grid_for(p->n_groups, kCostThreads / 32, (uint32_t)sm_count * 8u);
  switch (pass) {
    case 0: {
      const uint32_t n = p->n_keys > p->n_nodes ? p->n_keys : p->n_nodes;
      drain_budget_keys_init_kernel<<<grid_for(n, 256, (uint32_t)sm_count * 4u), 256, 0, s>>>(a, p->occupancy, p->n_keys);
      if (p->n_groups) drain_budget_walk_kernel<false><<<walk_grid, kCostThreads, 0, s>>>(a);
      return launch_result(p->n_groups ? 2 : 1);
    }
    case 1:
      drain_budget_walk_kernel<true><<<walk_grid, kCostThreads, 0, s>>>(a);
      drain_budget_finish_kernel<<<grid_for((uint64_t)p->table_mask + 1, 256, (uint32_t)sm_count * 8u), 256, 0, s>>>(a);
      return launch_result(2);
    default:  // the table alone, for the DS drain's per-key form
      drain_budget_walk_kernel<true><<<walk_grid, kCostThreads, 0, s>>>(a);
      return launch_result(1);
  }
}

int launch_drain_restart_pairs(const DrainBudgetCostLaunch* p, unsigned long long* pairs, uint32_t capacity, int sm_count,
                               cudaStream_t s) {
  if (p->n_groups == 0) return 0;
  const DrainBudgetCostArgs a{p->lws, p->lws_out, p->groups, p->pod_state, p->pod_ident, p->baseline,
                              p->by_domain ? p->nodes : nullptr, nullptr, pairs, nullptr, p->counts,
                              p->n_pods, p->n_lws, p->n_groups, p->n_nodes, p->n_domains, capacity};
  drain_budget_walk_kernel<false, true>
      <<<grid_for(p->n_groups, kCostThreads / 32, (uint32_t)sm_count * 8u), kCostThreads, 0, s>>>(a);
  return launch_result(1);
}

// --------------------------------------------------------------------------
// DS drain (lwse_resident_ds_drain*): the definitions are in lwse.h
// --------------------------------------------------------------------------
//   ds_drain_lost_kernel     the set form: one warp per LWS row over its group range (as drain_budget_kernel),
//                            lost[L] and the after copy of its lws_out row (ready_replicas - lost, clamped).
//   ds_drain_pairs_kernel    the per-key form: (row, key) pairs = the linked rows of L summed over the (LWS, key)
//                            entries with lost > 0.
//   ds_drain_insert_kernel   one thread per (LWS, key) entry with lost > 0, over the rows linked to L: the key
//                            row's rows_touched / rows_zeroed, and the row's facts ORed into the (DS, key) table.
//   ds_drain_finish_kernel   every (DS, key) entry gated by the DS's before flags into its key's DS columns.
struct DsDrainLostArgs {
  const lwse_lws_rec* lws;
  const lwse_lws_out* lws_out;
  const lwse_group_rec* groups;
  const lwse_group_out* before;
  const lwse_group_out* after;
  uint32_t* lost;
  lwse_lws_out* lws_after;
  uint32_t n_lws, n_groups;
};

__global__ void __launch_bounds__(256) ds_drain_lost_kernel(const DsDrainLostArgs a) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t n_warps = gridDim.x * (blockDim.x / 32);
  for (uint32_t L = (blockIdx.x * blockDim.x + threadIdx.x) / 32; L < a.n_lws; L += n_warps) {
    const uint4 r3 = ldg_cached(reinterpret_cast<const uint4*>(a.lws + L) + 3);
    const uint32_t gbase = r3.z, gcount = (uint64_t)r3.z + r3.w <= a.n_groups ? r3.w : 0u;
    uint32_t lost = 0;
    for (uint32_t i = lane; i < gcount; i += 32) {
      const uint32_t g = gbase + i;
      if (__ldg(&a.groups[g].lws_index) != L) continue;
      const uint32_t o = __ldcg(&a.before[g].flags), v = __ldcg(&a.after[g].flags);
      lost += (!(o & kRestartBits) && (v & kRestartBits) && (o & LWSE_GOUT_COND_READY)) ? 1u : 0u;
    }
    lost = __reduce_add_sync(0xFFFFFFFFu, lost);
    if (lane > 1) continue;
    const uint4* src = reinterpret_cast<const uint4*>(a.lws_out + L);
    uint4 v = __ldg(src + lane);
    if (lane == 0) {
      a.lost[L] = lost;
      v.w = (uint32_t)clamp_i32((int64_t)(int32_t)v.w - lost);  // ready_replicas
    }
    reinterpret_cast<uint4*>(a.lws_after + L)[lane] = v;
  }
}

int launch_ds_drain_lost(const lwse_lws_rec* d_lws, const lwse_lws_out* d_lws_out, uint32_t n_lws, const lwse_group_rec* d_groups,
                         const lwse_group_out* d_before, const lwse_group_out* d_after, uint32_t n_groups, uint32_t* d_lost,
                         lwse_lws_out* d_lws_after, int sm_count, cudaStream_t s) {
  if (n_lws == 0) return 0;
  const DsDrainLostArgs a{d_lws, d_lws_out, d_groups, d_before, d_after, d_lost, d_lws_after, n_lws, n_groups};
  ds_drain_lost_kernel<<<grid_for(n_lws, 256 / 32, (uint32_t)sm_count * 8u), 256, 0, s>>>(a);
  return launch_result(1);
}

constexpr uint32_t kDsdNewZeroed = 1u << 0;   // a spec row of the new revision falls below 1 ready
constexpr uint32_t kDsdNewChanged = 1u << 1;  // a spec row of the new revision changes its ready count

__global__ void __launch_bounds__(256) ds_drain_pairs_kernel(const DsDrainCostLaunch p) {
  unsigned long long pairs = 0;
  for (uint32_t h = blockIdx.x * blockDim.x + threadIdx.x; h <= p.lws_mask; h += gridDim.x * blockDim.x) {
    const unsigned long long k = __ldg(p.lws_keys + h);
    if (k == kEmptyKey || __ldg(&p.lws_vals[h].y) == 0) continue;
    const uint32_t L = (uint32_t)(k >> 32);
    pairs += __ldg(p.first + L + 1) - __ldg(p.first + L);
  }
  pairs = warp_sum_u64(pairs);
  if ((threadIdx.x & 31u) == 0 && pairs) atomicAdd(reinterpret_cast<unsigned long long*>(p.counts), pairs);
}

__global__ void __launch_bounds__(256) ds_drain_insert_kernel(const DsDrainCostLaunch p) {
  for (uint32_t h = blockIdx.x * blockDim.x + threadIdx.x; h <= p.lws_mask; h += gridDim.x * blockDim.x) {
    const unsigned long long k = __ldg(p.lws_keys + h);
    if (k == kEmptyKey) continue;
    const uint32_t lost = __ldg(&p.lws_vals[h].y);
    if (lost == 0) continue;
    const uint32_t L = (uint32_t)(k >> 32), key = (uint32_t)k;
    uint32_t touched = 0, zeroed = 0;
    for (uint32_t j = __ldg(p.first + L), end = __ldg(p.first + L + 1); j < end; j++) {
      const uint4 e = __ldg(p.entries + j);  // {DS row, slot | spec, ready_before, 0}
      const int32_t rb = (int32_t)e.z, ra = clamp_i32((int64_t)rb - lost);
      const bool zero = rb >= 1 && ra < 1;
      touched++;
      zeroed += zero ? 1u : 0u;
      uint32_t bits = 0, old_mask = 0;
      if (e.y & kDsDrainSpec) {
        const uint32_t slot = e.y & 0xFFu;
        if (slot == kDsDrainNewSlot)
          bits = (zero ? kDsdNewZeroed : 0u) | (ra != rb ? kDsdNewChanged : 0u);
        else if (zero)
          old_mask = 1u << slot;
      }
      const unsigned long long dk = (unsigned long long)e.x << 32 | key;
      uint32_t t = table_slot(dk, p.table_mask);
      bool placed = false;
      for (uint32_t probe = 0; probe <= p.table_mask; probe++, t = (t + 1u) & p.table_mask) {
        const unsigned long long prev = atomicCAS(p.keys + t, kEmptyKey, dk);
        if (prev == kEmptyKey || prev == dk) {
          if (bits) atomicOr(&p.vals[t].x, bits);
          if (old_mask) atomicOr(&p.vals[t].y, old_mask);
          placed = true;
          break;
        }
      }
      if (!placed) atomicAdd(p.counts + 2, 1u);  // full: the call fails
    }
    atomicAdd(&p.cost[key].rows_touched, touched);
    if (zeroed) atomicAdd(&p.cost[key].rows_zeroed, zeroed);
  }
}

__global__ void __launch_bounds__(256) ds_drain_finish_kernel(const DsDrainCostLaunch p) {
  for (uint32_t h = blockIdx.x * blockDim.x + threadIdx.x; h <= p.table_mask; h += gridDim.x * blockDim.x) {
    const unsigned long long k = p.keys[h];
    if (k == kEmptyKey) continue;
    const uint32_t d = (uint32_t)(k >> 32), key = (uint32_t)k;
    const uint2 v = p.vals[h];
    const uint4 b = __ldg(reinterpret_cast<const uint4*>(p.before + d));  // {flags, drained_revs, ready_revs, 0}
    lwse_ds_drain_cost* c = p.cost + key;
    atomicAdd(&c->ds_touched, 1u);
    if ((v.x & kDsdNewZeroed) && (b.x & LWSE_DOUT_NEW_READY)) atomicAdd(&c->ds_service_lost, 1u);
    if (v.y & b.z) atomicAdd(&c->ds_old_service_lost, 1u);
    if ((v.x & kDsdNewChanged) && (b.x & LWSE_DOUT_STABLE)) atomicAdd(&c->ds_stalled, 1u);
  }
}

int launch_ds_drain_cost(const DsDrainCostLaunch* p, int pass, int sm_count, cudaStream_t s) {
  const unsigned lws_grid = grid_for((uint64_t)p->lws_mask + 1, 256, (uint32_t)sm_count * 8u);
  if (pass == 0) {
    ds_drain_pairs_kernel<<<lws_grid, 256, 0, s>>>(*p);
    return launch_result(1);
  }
  ds_drain_insert_kernel<<<lws_grid, 256, 0, s>>>(*p);
  ds_drain_finish_kernel<<<grid_for((uint64_t)p->table_mask + 1, 256, (uint32_t)sm_count * 8u), 256, 0, s>>>(*p);
  return launch_result(2);
}

}  // namespace lwse
