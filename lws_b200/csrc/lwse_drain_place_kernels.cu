// Drain placement (lwse_resident_drain_place_cost, sm_90a); the definition is in lwse.h, the locality rule's
// argument in DESIGN.md §3.5.
//
//   drain_place_dom_free_kernel   a warp per domain: its free slots over the node index (rule (b) reads them).
//   drain_place_prep_kernel    a thread per request row: the baseline's PLACED / UNSCHEDULABLE / CONFLICT totals,
//                              the restart pairs (the sum of the drain budget's groups_restarted over the keys),
//                              pinned rows counted per group (the group -> request index) and under the key of
//                              their leader's node (U_k's first source), and the rule-(b) items counted.
//   drain_place_group_fill_kernel   the group -> pinned request index, by cursor (after the scan).
//   drain_place_unpin_kernel   a thread per restart pair (key, group) over the group's pinned requests whose leader
//                              is not on the key (U_k's second source; the first already holds the others):
//                              counted, or, after the scan, filled — with the first source's rows — into u_rows.
//   drain_place_rows_kernel    every key row started: groups_restarted, |U_k|, the baseline totals.
//   drain_place_items_kernel   the deduplicated (key, namespace) items: rule (a) from u_rows (with the rows of no
//                              namespace counted straight into their key rows), rule (b) from the baseline rows;
//                              then the drain instance of place_ns_kernel solves them.
#include "lwse_device.cuh"
#include "lwse_launch.cuh"

namespace lwse {

constexpr unsigned long long kFreeItem = ~0ull;

// The key whose drain set holds node n: the node itself, or its domain (by domain_id alone); LWSE_NONE for none.
__device__ __forceinline__ uint32_t place_key_of(const DrainPlaceLaunch& p, uint32_t n) {
  if (n >= p.n_nodes) return LWSE_NONE;
  if (!p.by_domain) return n;
  const uint32_t d = __ldg(&p.nodes[n].domain_id);
  return d < p.n_domains ? d : LWSE_NONE;
}

__device__ __forceinline__ uint32_t node_free(const DrainPlaceLaunch& p, uint32_t n) {
  const uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(p.nodes + n) + 3);  // capacity | flags << 16
  const uint32_t cap = w & 0xFFFFu, occ = p.occupancy ? __ldg(p.occupancy + n) : 0u;
  return cap > occ ? cap - occ : 0u;
}

__device__ __forceinline__ void insert_item(const DrainPlaceLaunch& p, uint32_t key, uint32_t ns) {
  const unsigned long long k = (unsigned long long)key << 32 | ns;
  unsigned long long h = k ^ (k >> 33);
  h *= 0xFF51AFD7ED558CCDull;
  h ^= h >> 33;
  uint32_t t = (uint32_t)h & p.item_mask;
  for (uint32_t probe = 0; probe <= p.item_mask; probe++, t = (t + 1u) & p.item_mask) {
    const unsigned long long prev = atomicCAS(p.item_keys + t, kFreeItem, k);
    if (prev == k) return;
    if (prev == kFreeItem) {
      const uint32_t at = atomicAdd(p.counts + 4, 1u);
      if (at < p.item_capacity) p.items[at] = make_uint2(key, ns);
      else atomicAdd(p.counts + 5, 1u);
      return;
    }
  }
  atomicAdd(p.counts + 5, 1u);  // full: the call fails
}

// Rule (b) for request row r: a row that is not pinned, PLACED in domain d of the baseline, is an item of its
// namespace for the key d (domain scope), or for its chosen node and every usable node n of d with
// dom_free[d] - free[n] < size (node scope).  Returns the items (emit = false) or inserts them.
template <bool kEmit>
__device__ __forceinline__ uint32_t rule_b(const DrainPlaceLaunch& p, uint32_t r) {
  const uint4 hi = __ldg(reinterpret_cast<const uint4*>(p.reqs + r) + 1);  // {group, ns, size, leader_node}
  if (hi.w != LWSE_NONE || hi.y >= p.n_namespaces) return 0u;
  const uint4 o = __ldg(reinterpret_cast<const uint4*>(p.base + r));
  if (!(o.z & LWSE_PLACE_PLACED) || o.x >= p.n_domains) return 0u;
  const uint32_t d = o.x, ns = hi.y;
  if (p.by_domain) {
    if (kEmit) insert_item(p, d, ns);
    return 1u;
  }
  uint32_t n_items = 0;
  if (o.y < p.n_nodes) {
    if (kEmit) insert_item(p, o.y, ns);
    n_items++;
  }
  const uint32_t f = __ldg(p.dom_first + d), l = __ldg(p.dom_first + d + 1u);
  const uint32_t dom_free = __ldcg(p.dom_free + d), size = hi.z;
  for (uint32_t i = f; i < l; i++) {
    const uint32_t n = __ldg(p.node_order + i);
    if (n == o.y || dom_free - node_free(p, n) >= size) continue;
    if (kEmit) insert_item(p, n, ns);
    n_items++;
  }
  return n_items;
}

// A warp per domain over its run of the node index: dom_free[d], the free slots the round's capacity vector holds.
__global__ void __launch_bounds__(256) drain_place_dom_free_kernel(const DrainPlaceLaunch p) {
  const uint32_t lane = threadIdx.x & 31u, n_warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t d = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; d < p.n_domains; d += n_warps) {
    uint32_t sum = 0;
    for (uint32_t i = __ldg(p.dom_first + d) + lane, l = __ldg(p.dom_first + d + 1u); i < l; i += 32u)
      sum += node_free(p, __ldg(p.node_order + i));
    sum = __reduce_add_sync(0xFFFFFFFFu, sum);
    if (lane == 0) p.dom_free[d] = sum;
  }
}

__global__ void __launch_bounds__(256) drain_place_prep_kernel(const DrainPlaceLaunch p) {
  const uint32_t lane = threadIdx.x & 31u, stride = gridDim.x * blockDim.x;
  uint32_t c[5] = {0u, 0u, 0u, 0u, 0u};
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < p.n_keys; k += stride)
    c[4] += __ldg(&p.cost[k].groups_restarted);  // every restart pair adds one to its key's count
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < p.n_reqs; r += stride) {
    const uint32_t f = __ldg(&p.base[r].flags);
    c[0] += (f & LWSE_PLACE_PLACED) ? 1u : 0u;
    c[1] += (f & LWSE_PLACE_UNSCHEDULABLE) ? 1u : 0u;
    c[2] += (f & LWSE_PLACE_CONFLICT) ? 1u : 0u;
    const uint4 hi = __ldg(reinterpret_cast<const uint4*>(p.reqs + r) + 1);
    if (hi.w != LWSE_NONE) {
      if (hi.x < p.n_groups) atomicAdd(p.g_count + hi.x, 1u);
      const uint32_t k = place_key_of(p, hi.w);
      if (k != LWSE_NONE) atomicAdd(p.u_count + k, 1u);
    }
    c[3] += rule_b<false>(p, r);
  }
#pragma unroll
  for (int k = 0; k < 5; k++) {
    const uint32_t sum = __reduce_add_sync(0xFFFFFFFFu, c[k]);
    if (lane == 0 && sum) atomicAdd(p.counts + (k < 4 ? k : 6), sum);
  }
}

__global__ void __launch_bounds__(256) drain_place_group_fill_kernel(const DrainPlaceLaunch p) {
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < p.n_reqs; r += gridDim.x * blockDim.x) {
    const uint4 hi = __ldg(reinterpret_cast<const uint4*>(p.reqs + r) + 1);
    if (hi.w != LWSE_NONE && hi.x < p.n_groups) p.g_reqs[atomicAdd(p.g_cursor + hi.x, 1u)] = r;
  }
}

// kFill = false: |U_k| from the restart pairs; true: u_rows from both sources.
template <bool kFill>
__global__ void __launch_bounds__(256) drain_place_unpin_kernel(const DrainPlaceLaunch p) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < p.n_pairs || (kFill && i < p.n_reqs); i += stride) {
    if (kFill && i < p.n_reqs) {  // the rows whose leader is on the key
      const uint32_t leader = __ldg(&p.reqs[i].leader_node);
      const uint32_t k = leader != LWSE_NONE ? place_key_of(p, leader) : LWSE_NONE;
      if (k != LWSE_NONE) p.u_rows[atomicAdd(p.u_cursor + k, 1u)] = i;
    }
    if (i >= p.n_pairs) continue;
    const unsigned long long pr = __ldg(p.pairs + i);
    const uint32_t k = (uint32_t)(pr >> 32), g = (uint32_t)pr;
    for (uint32_t j = __ldcg(p.g_first + g), end = __ldcg(p.g_first + g + 1u); j < end; j++) {
      const uint32_t r = __ldcg(p.g_reqs + j);
      if (place_key_of(p, __ldg(&p.reqs[r].leader_node)) == k) continue;  // (the first source holds it)
      if (kFill) p.u_rows[atomicAdd(p.u_cursor + k, 1u)] = r;
      else atomicAdd(p.u_count + k, 1u);
    }
  }
}

__global__ void __launch_bounds__(256) drain_place_rows_kernel(const DrainPlaceLaunch p) {
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < p.n_keys; k += gridDim.x * blockDim.x) {
    uint4* row = reinterpret_cast<uint4*>(p.rows + k);
    const uint32_t u = __ldcg(p.u_first + k + 1u) - __ldcg(p.u_first + k);
    row[0] = make_uint4(__ldg(&p.cost[k].groups_restarted), u, 0u, 0u);
    row[1] = make_uint4(0u, 0u, 0u, 0u);
    row[2] = make_uint4(__ldcg(p.counts + 0), __ldcg(p.counts + 1), __ldcg(p.counts + 2), 0u);
    row[3] = make_uint4(0u, 0u, 0u, 0u);
  }
}

__global__ void __launch_bounds__(256) drain_place_items_kernel(const DrainPlaceLaunch p) {
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t n_unp = __ldcg(p.u_first + p.n_keys);
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n_unp || j < p.n_reqs; j += stride) {
    if (j < n_unp) {  // rule (a): the key of entry j is the last k with u_first[k] <= j
      uint32_t lo = 0, hi = p.n_keys;
      while (hi - lo > 1u) {
        const uint32_t mid = (lo + hi) >> 1;
        if (__ldcg(p.u_first + mid) <= j) lo = mid;
        else hi = mid;
      }
      const uint32_t r = __ldcg(p.u_rows + j), ns = __ldg(&p.reqs[r].ns);
      if (ns < p.n_namespaces) {
        insert_item(p, lo, ns);
      } else {  // no namespace: the round gives the unpinned row UNSCHEDULABLE without a solve
        uint32_t c[kDrainCounts] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
        drain_place_count(c, __ldg(reinterpret_cast<const uint4*>(p.base + r)),
                          make_uint4(LWSE_NONE, LWSE_NONE, LWSE_PLACE_UNSCHEDULABLE, 0u), true);
        uint32_t* krow = reinterpret_cast<uint32_t*>(p.rows + lo);
        for (uint32_t f = 0; f < kDrainCounts; f++)
          if (c[f]) atomicAdd(krow + 2u + f, c[f]);
      }
    }
    if (j < p.n_reqs) rule_b<true>(p, j);
  }
}

int launch_drain_place(const DrainPlaceLaunch* p, int pass, int sm_count, cudaStream_t s) {
  const unsigned req_grid = grid_for(p->n_reqs, 256, (uint32_t)sm_count * 8u);
  switch (pass) {
    case 0: {
      drain_place_dom_free_kernel<<<grid_for((uint64_t)p->n_domains * 32u, 256, (uint32_t)sm_count * 8u), 256, 0, s>>>(*p);
      drain_place_prep_kernel<<<req_grid, 256, 0, s>>>(*p);
      if (const int r = launch_result(2); r < 0) return r;
      if (const int r = launch_index_scan(p->g_count, p->g_first, p->g_cursor, p->n_groups, s); r < 0) return r;
      drain_place_group_fill_kernel<<<req_grid, 256, 0, s>>>(*p);
      return launch_result(4);
    }
    case 1: {
      drain_place_unpin_kernel<false><<<grid_for(p->n_pairs, 256, (uint32_t)sm_count * 8u), 256, 0, s>>>(*p);
      if (const int r = launch_result(1); r < 0) return r;
      if (const int r = launch_index_scan(p->u_count, p->u_first, p->u_cursor, p->n_keys, s); r < 0) return r;
      return 2;
    }
    default: {
      const uint64_t n = p->n_pairs > p->n_reqs ? p->n_pairs : p->n_reqs;
      drain_place_unpin_kernel<true><<<grid_for(n, 256, (uint32_t)sm_count * 8u), 256, 0, s>>>(*p);
      drain_place_rows_kernel<<<grid_for(p->n_keys, 256, (uint32_t)sm_count * 4u), 256, 0, s>>>(*p);
      drain_place_items_kernel<<<grid_for((uint64_t)(p->n_reqs > p->n_unpinned ? p->n_reqs : p->n_unpinned), 256, (uint32_t)sm_count * 8u), 256, 0, s>>>(*p);
      if (const int r = launch_result(3); r < 0) return r;
      const int solved = launch_place_ns_drain(p, sm_count, s);
      return solved < 0 ? solved : 3 + solved;
    }
  }
}

}  // namespace lwse
