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

static int launched_or_fail(int kernels, int* cuda_err) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    *cuda_err = (int)e;
    return -1;
  }
  return kernels;
}

static unsigned grid_for(uint64_t items, uint32_t per_cta, uint32_t cap) {
  uint64_t grid = (items + per_cta - 1) / per_cta;
  if (grid < 1) grid = 1;
  return (unsigned)(grid < cap ? grid : cap);
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
                      lwse_group_rec* d_groups, uint32_t n_groups, uint32_t* d_counts, int sm_count, cudaStream_t s,
                      int* cuda_err) {
  *cuda_err = 0;
  const DrainMarkArgs a{d_mask, d_ident, d_state, d_groups, d_counts, n_pods, n_groups, n_nodes};
  const uint64_t items = n_pods > n_groups ? n_pods : n_groups;
  drain_mark_kernel<<<grid_for(items, 256, (uint32_t)sm_count * 16u), 256, 0, s>>>(a);
  return launched_or_fail(1, cuda_err);
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
                      uint32_t capacity, uint32_t* d_counts, int sm_count, cudaStream_t s, int* cuda_err) {
  *cuda_err = 0;
  const DrainDiffArgs a{d_before, d_after, d_groups, d_rows, d_outs_before, d_outs_after, d_counts, capacity, n_groups};
  drain_diff_kernel<<<grid_for(n_groups, 256, (uint32_t)sm_count * 4u), 256, 0, s>>>(a);
  return launched_or_fail(1, cuda_err);
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
                      lwse_drain_cost* d_cost, uint32_t n_nodes, int sm_count, cudaStream_t s, int* cuda_err) {
  *cuda_err = 0;
  if (n_groups == 0) return 0;
  const DrainCostArgs a{d_lws, d_groups, d_state, d_ident, d_baseline, d_cost, n_pods, n_lws, n_groups, n_nodes};
  drain_cost_kernel<<<grid_for(n_groups, kCostThreads / 32, (uint32_t)sm_count * 8u), kCostThreads, 0, s>>>(a);
  return launched_or_fail(1, cuda_err);
}

}  // namespace lwse
