// Placement round, namespace-parallel form (sm_90a) — same build-defined spec as
// lwse_place_kernels.cu (oracle/lwse_oracle_place.c), for request tables GROUPED BY NAMESPACE.
//
// Exclusivity is per namespace and capacity is a snapshot that no claim consumes, so the
// namespaces are independent sub-problems.  That turns the round's hot state — the holder table
// of one namespace (8 B x domains), the per-domain free capacity and the condensed node-topology
// table (one word per usable node: free slots | domain, in domain order) — into a few tens of KB
// that fit the shared memory of ONE CTA:
//
//   place_condense_kernel   node rows + occupancy -> sorted node words + per-domain capacity
//                           (a warp per domain over its run of the domain-sorted node index:
//                           no atomics), and the namespace index of the request table
//                           (ns_first[v] = first request of namespace v; order violations counted).
//   place_ns_kernel         one CTA per namespace.  The capacities and the domain index are staged
//                           with cp.async.bulk + mbarrier (issued by one thread while the others
//                           clear the holder table and take the pinned claims), the holder table
//                           lives in shared memory, claims are 64-bit shared-memory atomicMin,
//                           rounds are separated by __syncthreads() — no grid or cluster barrier,
//                           no L2 round trip per domain.  Deferred acceptance runs to ITS OWN
//                           fixed point per namespace.
//     two-level form        512 threads.  After the pinned claims the CTA compacts the CANDIDATE
//                           domains — no pinned holder (a pinned key beats every unpinned key) and
//                           capacity left — into a list {domain, free}; the unpinned holder table
//                           is indexed by list position, so a (request, round) search is two
//                           coalesced shared-memory streams over the candidates (a fourth of the
//                           domains on C3) and one read of the chosen domain's (free | node) run.
//                           16 KB + 36 B per domain of shared memory: no staging of the node
//                           table, and the sweep kernels keep the SMs' shared memory.
//     scan form             256 threads; the node-word table and the node order are staged whole
//                           with TMA (cp.async.bulk.tensor.2d through a CUtensorMap + cp.async.bulk)
//                           and every (request x node) pair is scored from shared memory:
//                           feasibility + both rendezvous hashes per pair, lexicographic arg-max
//                           (domain score, lower domain, node score, lower node) — identical rows.
//   Inside a tick both forms also append the result rows that differ from the previous tick's to
//   the device change list (PlaceNsArgs::prev …) — no separate diff kernel.
//
// Indexed form — a request table NOT grouped by namespace (a patch moved a request to another
// namespace): the namespace kernel reaches its requests through a namespace index,
// ns_rows[ns_first[v] .. ns_first[v+1]) = the request rows of namespace v, built on the device by
//   place_index_count_kernel   requests per namespace
//   place_index_scan_kernel    exclusive scan -> ns_first, per-namespace cursors
//   place_index_fill_kernel    ns_rows, by cursor
// The order inside a namespace is arbitrary and the result does not depend on it: keys carry the
// request ROW, pinned claims are atomicMin on those keys and the unpinned list is built with atomics
// anyway.  The index is rebuilt only when the namespace column changed; other calls reuse it.
#include <cuda.h>

#include <cstdlib>
#include <cstring>

#include "lwse_device.cuh"
#include "lwse_launch.cuh"

namespace lwse {

struct PlaceNsArgs {
  const lwse_node_rec* nodes;
  const lwse_place_req* reqs;  // grouped by namespace (ns non-decreasing), unless ns_rows is set
  const uint32_t* occupancy;   // nullable; n_parts blocks of n_nodes counters, part_stride_bytes apart
  lwse_place_out* out;
  const uint32_t* dom_first;   // the node index (node_index_*_kernel); dom_first[n_domains] = usable nodes
  const uint32_t* node_order;
  uint32_t* g_words;     // condensed node words in domain-sorted position, padded with zeros to whole rows of 256
  uint32_t* g_nodes2;    // the same positions: free slots (4 bits) | node index — the two-level form's level 2
  uint32_t* g_dom_free;  // n_domains (+ padding)
  uint32_t* ns_first;    // n_namespaces + 1
  uint32_t* unpinned;    // n_reqs: namespace v's live unpinned requests at [ns_first[v], …)
  // indexed form (null: the table is grouped and a position is a row)
  uint32_t* ns_rows;     // n_reqs: position -> request row
  uint32_t* ns_count;    // n_namespaces: requests per namespace (all zero between index builds)
  uint32_t* ns_cursor;   // n_namespaces: fill cursors
  uint32_t* counters;    // this call's block: [0] max rounds [1] live unpinned [2] order violations [3] (request, round) scans
  uint32_t* next_counters;  // the other block, cleared for the next call
  uint32_t n_nodes, n_domains, n_reqs, n_namespaces;
  uint32_t n_parts;
  uint64_t part_stride_bytes;
  uint32_t word_rows;   // rows of 256 words of g_words
  uint32_t scan;        // 1 = brute-force (request x node) form
  uint32_t stage_words; // the word table fits shared memory and is staged
  uint32_t use_tensor_map;
  // a tick's change list (all null / 0 = off): rows that differ from `prev` are appended, `prev` is updated
  lwse_place_out* prev;
  uint32_t* chg_rows;
  lwse_place_out* chg_outs;
  uint32_t* chg_count;
  uint32_t chg_capacity;
  // multi-rank ticks: `occupancy` is the base of the exchange buffers; the blocks to sum are those of
  // step (lagged ? step - 1 : step) where step = *xch_step (the push kernel right before stored it)
  const unsigned long long* xch_step;
  uint64_t xch_half_bytes;
  uint32_t xch_lagged;
};

// What the drain-placement instance of the namespace kernel reads besides PlaceNsArgs (lwse_resident_drain_place_cost).
// That instance stages no word table, so the view travels in the bytes of its tensor-map parameter, and
// PlaceNsArgs (with every other instance's code) stays as it is.  It runs over items (key, namespace) instead of
// namespaces; out / unpinned / marks are per-CTA slices of slice_rows entries indexed by the position inside the
// namespace, so that two CTAs may solve the same namespace for different keys at once.
struct DrainNsView {
  const uint2* items;            // {key, namespace}
  const uint32_t* n_items;       // device count of insertions (capped by item_capacity)
  uint32_t item_capacity;
  const uint32_t* u_first;       // [n_keys + 1]: U_k = u_rows[u_first[k] .. u_first[k + 1])
  const uint32_t* u_rows;
  const uint32_t* pos;           // request row -> position in the namespace index (ns_rows), LWSE_NONE outside
  uint8_t* marks;                // per CTA: 1 = the row at that position is in U_k
  const lwse_place_out* base;    // the baseline rows
  uint32_t* rows;                // the key rows (lwse_drain_place_cost, 16 words each)
  uint32_t slice_rows;           // the largest namespace
  uint32_t by_domain;
};
static_assert(sizeof(DrainNsView) <= sizeof(CUtensorMap), "the view travels in the tensor-map parameter");

// The set-overlay instance (lwse_resident_drain_place_waves): DrainNsView with items {column, namespace} of the
// current probe W_c ∪ {k}, `rows` the column rows and U_k read through u_first / u_rows at the key in state[0]; the
// wave state says what W_c already drains.
struct SetNsView {
  DrainNsView d;
  const uint32_t* state;                // [0] the key k of the current step
  const unsigned long long* u_wave;     // [n_reqs] bit c: the row is in U of wave c
  const unsigned long long* key_wave;   // [n_nodes] (node scope) or [n_domains] (domain scope) bit c: in wave c
  const uint32_t* drained;              // node scope: [64 * n_domains] free slots wave c drains from domain d
};
static_assert(sizeof(SetNsView) <= sizeof(CUtensorMap), "the view travels in the tensor-map parameter");

// The rollout instance (lwse_resident_rollout_place): DrainNsView's items {entry, namespace}, slices, baseline and
// rows (u_first, u_rows, pos, marks and by_domain unused); per entry its extra rows E_i after the namespace's
// resident rows.
struct RollNsView {
  DrainNsView d;
  const lwse_place_req* extra;  // every entry's E_i, entry i's at ent[i].x
  const uint4* ent;             // [entries] {first extra row, |E_i|, group_base, group_count}
  uint32_t n_resident;          // extra row j of an entry has row index (and key) n_resident + j
};
static_assert(sizeof(RollNsView) <= sizeof(CUtensorMap), "the view travels in the tensor-map parameter");

// The rollout wave instance (lwse_resident_rollout_place_waves): RollNsView with items {slot, namespace}; slot s
// probes column (ns, w) with key k: the extra rows of the ns entries already in wave w, in query order, then E_k.
struct RollWaveNsView {
  RollNsView r;
  const uint4* desc;  // [slots] {k, first list entry, list length, the column's extra rows}
  const uint4* col;   // the column lists: {E_j's first extra row, its offset in the column, group_base, group_count}
};
static_assert(sizeof(RollWaveNsView) <= sizeof(CUtensorMap), "the view travels in the tensor-map parameter");

// The rollout instance's counters, words 4..14 of the entry's lwse_rollout_place row: placed, stranded, own_lost,
// bumped, then the what-if counters (the three totals as deltas against the baseline).
constexpr uint32_t kRollCounts = 11;

__device__ __forceinline__ uint32_t mix32n(uint32_t x) {
  x ^= x >> 16;
  x *= 0x85EBCA6Bu;
  x ^= x >> 13;
  x *= 0xC2B2AE35u;
  x ^= x >> 16;
  return x;
}

__device__ __forceinline__ unsigned long long ns_place_key(unsigned long long priority, uint32_t index, bool pinned) {
  return ((unsigned long long)(pinned ? 0 : 1) << 63) | (((priority >> 25) & 0x7FFFFFFFFFull) << 24) |
         (unsigned long long)(index & 0xFFFFFFu);
}

__device__ __forceinline__ uint32_t occupancy_sum(const PlaceNsArgs& a, const uint32_t* base, uint32_t n) {
  if (!base) return 0u;
  uint32_t occ = 0;
  for (uint32_t p = 0; p < a.n_parts; p++)
    occ += ldg_keep_u32(reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint8_t*>(base) +
                                                           (uint64_t)p * a.part_stride_bytes) + n);
  return occ;
}

__device__ __forceinline__ void store_row(lwse_place_out* p, uint32_t d, uint32_t n, uint32_t flags, uint32_t score) {
  *reinterpret_cast<uint4*>(p) = make_uint4(d, n, flags, score);
}

// --------------------------------------------------------------------------
// condense: node words, domain capacities, namespace index
// --------------------------------------------------------------------------
__global__ void __launch_bounds__(256) place_condense_kernel(const PlaceNsArgs a) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t gwarp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t gtid = blockIdx.x * blockDim.x + threadIdx.x, gsize = gridDim.x * blockDim.x;
  pdl_launch_dependents();  // the namespace kernel may load its requests meanwhile; it waits before the tables below
  pdl_wait_prior();         // the previous call's namespace kernel may still read the tables written here
  const uint32_t* occ_base = a.occupancy;
  if (a.xch_step != nullptr && occ_base != nullptr) {
    const unsigned long long step = *reinterpret_cast<const volatile unsigned long long*>(a.xch_step);
    const unsigned long long read_step = (a.xch_lagged && step > 1ull) ? step - 1ull : step;
    occ_base = reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint8_t*>(occ_base) + (read_step % 3ull) * a.xch_half_bytes);
  }
  // A. a warp per domain: its nodes are a run of the sorted index
  for (uint32_t d = gwarp; d < a.n_domains; d += n_warps) {
    const uint32_t first = ldg_keep_u32(a.dom_first + d), last = ldg_keep_u32(a.dom_first + d + 1u);
    uint32_t sum = 0;
    for (uint32_t i = first + lane; i < last; i += 32u) {
      const uint32_t n = ldg_keep_u32(a.node_order + i);
      const uint4 nr = ldg_keep(reinterpret_cast<const uint4*>(a.nodes + n));
      const uint32_t cap = nr.w & 0xFFFFu, occ = occupancy_sum(a, occ_base, n);
      const uint32_t fr = cap > occ ? cap - occ : 0u;
      a.g_words[i] = (min(fr, 15u) << 28) | d;
      a.g_nodes2[i] = (min(fr, 15u) << 28) | n;
      sum += fr;
    }
    sum = __reduce_add_sync(0xFFFFFFFFu, sum);
    if (lane == 0) a.g_dom_free[d] = sum;
  }
  // B. the namespace index of the (promised) grouped request table; the indexed form has its own
  const bool grouped = a.ns_rows == nullptr;
  if (grouped && a.n_reqs == 0u) {
    for (uint32_t v = gtid; v <= a.n_namespaces; v += gsize) a.ns_first[v] = 0u;
  }
  for (uint32_t i = gtid; i < a.n_reqs; i += gsize) {
    const uint4 hi = ldg_keep(reinterpret_cast<const uint4*>(a.reqs + i) + 1);
    const uint32_t b = hi.y;
    if (grouped) {
      uint32_t lo_v;  // namespaces (lo_v, b] start at request i; for i == 0 also namespace lo_v itself
      if (i == 0u) {
        for (uint32_t v = 0; v <= min(b, a.n_namespaces); v++) a.ns_first[v] = 0u;
      } else {
        const uint32_t prev = ldg_keep_u32(reinterpret_cast<const uint32_t*>(a.reqs + i - 1) + 5);  // .ns
        if (prev > b) atomicAdd(a.counters + 2, 1u);  // not grouped: the caller broke its promise
        lo_v = min(prev, a.n_namespaces);
        for (uint32_t v = lo_v + 1u; v <= min(b, a.n_namespaces); v++) a.ns_first[v] = i;
      }
      if (i == a.n_reqs - 1u)
        for (uint32_t v = min(b, a.n_namespaces) + 1u; v <= a.n_namespaces; v++) a.ns_first[v] = a.n_reqs;
    }
    if (b >= a.n_namespaces) {  // no such namespace: never takes part in a round
      const bool pinned = hi.w != LWSE_NONE;
      const uint4 row = make_uint4(LWSE_NONE, pinned ? hi.w : LWSE_NONE, (pinned ? LWSE_PLACE_PINNED : 0u) | LWSE_PLACE_UNSCHEDULABLE, 0u);
      *reinterpret_cast<uint4*>(a.out + i) = row;
      if (a.prev != nullptr) {
        const uint4 o = __ldcg(reinterpret_cast<const uint4*>(a.prev + i));
        if (row.x != o.x || row.y != o.y || row.z != o.z || row.w != o.w) {
          const uint32_t k = atomicAdd(a.chg_count, 1u);
          if (k < a.chg_capacity) {
            a.chg_rows[k] = i;
            *reinterpret_cast<uint4*>(a.chg_outs + k) = row;
          }
          *reinterpret_cast<uint4*>(a.prev + i) = row;
        }
      }
    }
  }
  if (gtid < 8u && a.next_counters != nullptr) a.next_counters[gtid] = 0u;
}

// --------------------------------------------------------------------------
// the namespace index of an ungrouped request table (indexed form)
// --------------------------------------------------------------------------
// A warp looks at 32 consecutive rows and takes one atomic per namespace among them
// (__match_any_sync): an ungrouped table is still mostly runs of one namespace.  Rows whose
// namespace does not exist are left out (the condense kernel marks them UNSCHEDULABLE).
__device__ __forceinline__ uint32_t index_ns_of(const PlaceNsArgs& a, uint32_t i) {
  if (i >= a.n_reqs) return LWSE_NONE;
  const uint32_t v = ldg_keep_u32(reinterpret_cast<const uint32_t*>(a.reqs + i) + 5);  // .ns
  return v < a.n_namespaces ? v : LWSE_NONE;
}

__global__ void __launch_bounds__(256) place_index_count_kernel(const PlaceNsArgs a) {
  pdl_launch_dependents();
  pdl_wait_prior();  // the request table a tick's scatter patched; the previous call's readers of the index
  const uint32_t lane = threadIdx.x & 31u, stride = gridDim.x * blockDim.x;
  for (uint32_t base = (blockIdx.x * blockDim.x + threadIdx.x) & ~31u; base < a.n_reqs; base += stride) {
    const uint32_t v = index_ns_of(a, base + lane);
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, v);
    if (v != LWSE_NONE && lane == (uint32_t)__ffs(peers) - 1u) atomicAdd(a.ns_count + v, (uint32_t)__popc(peers));
  }
}

// one CTA: first = exclusive scan of the counts (first[n] = the total), the cursors start there, the
// counts go back to zero.  Shared by the namespace index (per namespace) and the node index (per domain).
struct IndexScanArgs {
  uint32_t* count;
  uint32_t* first;
  uint32_t* cursor;
  uint32_t n;
};
constexpr uint32_t kIndexScanThreads = 1024;
__global__ void __launch_bounds__(kIndexScanThreads) place_index_scan_kernel(const IndexScanArgs a) {
  __shared__ uint32_t s_warp[32], s_carry;
  pdl_launch_dependents();
  pdl_wait_prior();
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  if (tid == 0) s_carry = 0u;
  __syncthreads();
  for (uint32_t base = 0; base < a.n; base += kIndexScanThreads) {
    const uint32_t v = base + tid;
    const uint32_t c = v < a.n ? __ldcg(a.count + v) : 0u;
    uint32_t x = c;  // inclusive scan inside the warp
#pragma unroll
    for (uint32_t o = 1; o < 32u; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31u) s_warp[warp] = x;
    __syncthreads();
    if (warp == 0) {
      uint32_t w = s_warp[lane];
#pragma unroll
      for (uint32_t o = 1; o < 32u; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, w, o);
        if (lane >= o) w += y;
      }
      s_warp[lane] = w;
    }
    __syncthreads();
    const uint32_t first = s_carry + (warp ? s_warp[warp - 1u] : 0u) + x - c;
    if (v < a.n) {
      a.first[v] = first;
      a.cursor[v] = first;
      a.count[v] = 0u;
    }
    __syncthreads();  // everybody has read s_carry and s_warp
    if (tid == kIndexScanThreads - 1u) s_carry = first + c;
    __syncthreads();
  }
  if (tid == 0) a.first[a.n] = s_carry;
}

__global__ void __launch_bounds__(256) place_index_fill_kernel(const PlaceNsArgs a) {
  pdl_launch_dependents();
  pdl_wait_prior();
  const uint32_t lane = threadIdx.x & 31u, stride = gridDim.x * blockDim.x;
  for (uint32_t base = (blockIdx.x * blockDim.x + threadIdx.x) & ~31u; base < a.n_reqs; base += stride) {
    const uint32_t i = base + lane, v = index_ns_of(a, i);
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, v);
    const uint32_t leader = (uint32_t)__ffs(peers) - 1u;
    uint32_t pos = 0;
    if (v != LWSE_NONE && lane == leader) pos = atomicAdd(a.ns_cursor + v, (uint32_t)__popc(peers));
    pos = __shfl_sync(0xFFFFFFFFu, pos, (int)leader);
    if (v != LWSE_NONE) a.ns_rows[pos + (uint32_t)__popc(peers & ((1u << lane) - 1u))] = i;
  }
}

// --------------------------------------------------------------------------
// the domain-sorted node index every placement form reads (lwse_upload_nodes, node-row patches)
// --------------------------------------------------------------------------
// dom_first[d] .. dom_first[d + 1] is the run of domain d in node_order, dom_first[n_domains] the
// number of usable nodes (schedulable, labelled, domain_id < n_domains); node_pos is the inverse of
// node_order, LWSE_NONE for a node no request can use.  The same count / scan / fill as the
// namespace index: the order inside a run is arbitrary, and every form breaks node ties by row.
struct NodeIndexArgs {
  const lwse_node_rec* nodes;
  uint32_t* dom_count;   // n_domains: nodes per domain (all zero between builds)
  uint32_t* dom_cursor;  // n_domains: fill cursors
  uint32_t* dom_first;   // n_domains + 1
  uint32_t* node_order;
  uint32_t* node_pos;
  uint32_t n_nodes, n_domains;
};

__device__ __forceinline__ uint32_t index_domain_of(const NodeIndexArgs& a, uint32_t n) {
  if (n >= a.n_nodes) return LWSE_NONE;
  const uint4 nr = __ldcg(reinterpret_cast<const uint4*>(a.nodes + n));  // (rows a tick's scatter just patched)
  const uint32_t flags = nr.w >> 16;
  const bool usable = (flags & LWSE_NODE_SCHEDULABLE) && (flags & LWSE_NODE_HAS_TOPOLOGY) && nr.z < a.n_domains;
  return usable ? nr.z : LWSE_NONE;
}

__global__ void __launch_bounds__(256) node_index_count_kernel(const NodeIndexArgs a) {
  pdl_launch_dependents();
  pdl_wait_prior();  // the node rows a tick's scatter patched; the previous round's readers of the index
  const uint32_t lane = threadIdx.x & 31u, stride = gridDim.x * blockDim.x;
  for (uint32_t base = (blockIdx.x * blockDim.x + threadIdx.x) & ~31u; base < a.n_nodes; base += stride) {
    const uint32_t d = index_domain_of(a, base + lane);
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, d);
    if (d != LWSE_NONE && lane == (uint32_t)__ffs(peers) - 1u) atomicAdd(a.dom_count + d, (uint32_t)__popc(peers));
  }
}

__global__ void __launch_bounds__(256) node_index_fill_kernel(const NodeIndexArgs a) {
  pdl_launch_dependents();
  pdl_wait_prior();
  const uint32_t lane = threadIdx.x & 31u, stride = gridDim.x * blockDim.x;
  for (uint32_t base = (blockIdx.x * blockDim.x + threadIdx.x) & ~31u; base < a.n_nodes; base += stride) {
    const uint32_t n = base + lane, d = index_domain_of(a, n);
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, d);
    const uint32_t leader = (uint32_t)__ffs(peers) - 1u;
    uint32_t pos = 0;
    if (d != LWSE_NONE && lane == leader) pos = atomicAdd(a.dom_cursor + d, (uint32_t)__popc(peers));
    pos = __shfl_sync(0xFFFFFFFFu, pos, (int)leader);
    if (n < a.n_nodes) {
      if (d != LWSE_NONE) {
        pos += (uint32_t)__popc(peers & ((1u << lane) - 1u));
        a.node_order[pos] = n;
        a.node_pos[n] = pos;
      } else {
        a.node_pos[n] = LWSE_NONE;
      }
    }
  }
}

size_t node_index_scratch_bytes(uint32_t n_domains) { return (size_t)n_domains * 8u + 16u; }

// count -> scan -> fill on `s`.  `scratch` (node_index_scratch_bytes) must be zero before the first build;
// every build leaves it zero again.  `pdl`: the predecessor on `s` is a kernel.
int launch_node_index(const lwse_node_rec* d_nodes, uint32_t n_nodes, uint32_t n_domains, uint32_t* d_dom_first,
                      uint32_t* d_node_order, uint32_t* d_node_pos, void* d_scratch, int sm_count, cudaStream_t s,
                      bool pdl) {
  NodeIndexArgs a{};
  a.nodes = d_nodes;
  a.dom_count = static_cast<uint32_t*>(d_scratch);
  a.dom_cursor = a.dom_count + n_domains;
  a.dom_first = d_dom_first;
  a.node_order = d_node_order;
  a.node_pos = d_node_pos;
  a.n_nodes = n_nodes;
  a.n_domains = n_domains;
  uint64_t grid = ((uint64_t)n_nodes + 255) / 256;
  if (grid < 1) grid = 1;
  if (grid > (uint64_t)sm_count * 8u) grid = (uint64_t)sm_count * 8u;
  cudaError_t e = launch_pdl(node_index_count_kernel, dim3((unsigned)grid), dim3(256), 0, s, pdl, a);
  if (e == cudaSuccess)
    e = launch_pdl(place_index_scan_kernel, dim3(1), dim3(kIndexScanThreads), 0, s, true,
                   IndexScanArgs{a.dom_count, a.dom_first, a.dom_cursor, n_domains});
  if (e == cudaSuccess) e = launch_pdl(node_index_fill_kernel, dim3((unsigned)grid), dim3(256), 0, s, true, a);
  if (e != cudaSuccess) return -(int)e;
  return 3;
}

// --------------------------------------------------------------------------
// one CTA per namespace
// --------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

constexpr uint32_t kNsScanThreads = 256;  // scan form: two CTAs (2 x ~100 KB of staged tables) share an SM
constexpr uint32_t kNsThreads = 512;      // two-level form: 16 warps, a warp per unpinned request and round
constexpr uint32_t kNsKeep = 2;           // requests per thread kept in registers between the claim and the result pass
constexpr uint32_t kNsCache = 256;        // unpinned requests of a namespace whose state lives in shared memory

// An unpinned request across the rounds (shared memory; written by the one warp that owns it).
// cur: what it proposed to last — a domain (scan form) or a candidate slot (two-level form).
struct NsReq {
  unsigned long long key;
  uint32_t r, key_lo, key_hi, size, cur, dead;
};

__device__ __forceinline__ void mbar_wait(unsigned long long* mbar) {
  uint32_t done = 0;
  while (!done)
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0; selp.u32 %0, 1, 0, p; }"
                 : "=r"(done) : "r"(smem_u32(mbar)) : "memory");
}

__device__ __forceinline__ void bulk_load(void* smem_dst, const void* gmem_src, uint32_t bytes, unsigned long long* mbar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(mbar))
               : "memory");
}

// A tick's change list: a result row that differs from the previous tick's is appended (and the
// previous-tick copy brought up to date) by the thread that produced it.
__device__ __forceinline__ void diff_row(const PlaceNsArgs& a, uint32_t r, const uint4 v) {
  if (a.prev == nullptr) return;
  const uint4 o = __ldcg(reinterpret_cast<const uint4*>(a.prev + r));
  if (v.x != o.x || v.y != o.y || v.z != o.z || v.w != o.w) {
    const uint32_t i = atomicAdd(a.chg_count, 1u);
    if (i < a.chg_capacity) {
      a.chg_rows[i] = r;
      *reinterpret_cast<uint4*>(a.chg_outs + i) = v;
    }
    *reinterpret_cast<uint4*>(a.prev + r) = v;
  }
}

// kIndexed: the requests of a namespace are reached through the index (ns_rows); results, keys and the
// unpinned list carry the request ROW either way.
// kDrain (two-level, indexed): the drain-placement instance.  A persistent grid over DrainNsView::items; per item
// the CTA lowers the staged capacity of the drained domain (a domain key: to 0; a node key: by the node's free
// slots, and level 2 skips the node's word), reads the rows of U_k as unpinned, keeps every result and the
// overflow state in its own slice (indexed by position, not row), diffs the namespace's rows against the
// baseline and adds the counts to the key's row.  The rows keep their keys (priority, ROW).
// kSet (with kDrain): the set-overlay instance.  Item {c, ns} solves ns for the probe W_c ∪ {k}: the staged
// capacities are rebuilt from the resident ones minus what the column drains (every domain of W_c and k zeroed, or
// every domain lowered by the free slots of its drained nodes), level 2 skips every drained node, and U_{W_c} ∪ U_k
// read as unpinned; the namespace's diff goes to column c's row.
// kRoll (with kDrain): the rollout instance.  Item {i, ns} solves ns with entry i's extra rows E_i: positions run over
// the namespace's resident rows through the index, then over E_i's rows (row index n_resident + j); nothing is
// lowered or unpinned; the namespace's diff goes to entry i's row.
// kWave (with kRoll): the rollout wave instance.  Item {s, ns} solves ns with the column's extra rows then E_k
// (RollWaveNsView); extra position q has row index n_resident + q; a resident row lost counts as own when its
// group lies in the range of k or of a listed entry; the namespace's diff goes to slot s's row.
template <bool kScan, bool kIndexed, bool kDrain = false, bool kSet = false, bool kRoll = false, bool kWave = false>
__global__ void __launch_bounds__(kScan ? kNsScanThreads : kNsThreads, 2)
    place_ns_kernel(const PlaceNsArgs a, const __grid_constant__ CUtensorMap words_map) {
  extern __shared__ uint8_t s_dyn[];
  // layout (from a 128-byte aligned base: the TMA destination):
  //   scan form, when they fit:  [words: word_rows x 256 u32] [node order: word_rows x 256 u32]
  //   [dom_free: n_domains u32] [dom_first: n_domains + 1 u32] [holder by domain: n_domains u64]
  //   two-level form:            [candidates: n_domains x {domain, free}] [holder by candidate: n_domains u64]
  //                              [slot of domain: n_domains u32]
  //   [request cache: kNsCache x 32 B] [mbarrier]
  uint8_t* s_raw = s_dyn + ((128u - (smem_u32(s_dyn) & 127u)) & 127u);
  const uint32_t table_bytes = (kScan && a.stage_words) ? a.word_rows * 1024u : 0u;
  const uint32_t free_bytes = ((a.n_domains * 4u) + 15u) & ~15u;
  const uint32_t first_bytes = (((a.n_domains + 1u) * 4u) + 15u) & ~15u;
  uint32_t* s_words = reinterpret_cast<uint32_t*>(s_raw);
  uint32_t* s_order = reinterpret_cast<uint32_t*>(s_raw + table_bytes);
  uint32_t* s_free = reinterpret_cast<uint32_t*>(s_raw + 2u * table_bytes);
  uint32_t* s_first = reinterpret_cast<uint32_t*>(s_raw + 2u * table_bytes + free_bytes);
  unsigned long long* s_hold = reinterpret_cast<unsigned long long*>(s_raw + 2u * table_bytes + free_bytes + first_bytes);
  uint2* s_cand = reinterpret_cast<uint2*>(s_hold + a.n_domains);
  unsigned long long* s_holdc = reinterpret_cast<unsigned long long*>(s_cand + (kScan ? 0u : a.n_domains));
  uint32_t* s_slot = reinterpret_cast<uint32_t*>(s_holdc + (kScan ? 0u : a.n_domains));
  NsReq* s_req = reinterpret_cast<NsReq*>(reinterpret_cast<uint8_t*>(s_slot) + (kScan ? 0u : free_bytes));
  unsigned long long* s_mbar = reinterpret_cast<unsigned long long*>(s_req + kNsCache);
  __shared__ uint32_t s_n_unp, s_n_cand, s_unsettled[3];
  // kDrain: the view travels in the tensor-map parameter's bytes (launch_place_ns_drain).  That instance must never
  // stage a word table (it would read the view as a tensor map): the two-level form stages none.
  static_assert(!(kDrain && kScan), "the drain instance is two-level: its tensor-map parameter holds the view");
  const DrainNsView* const drain = reinterpret_cast<const DrainNsView*>(&words_map);
  const SetNsView* const set = reinterpret_cast<const SetNsView*>(&words_map);
  static_assert(!kSet || kDrain, "the set instance is a drain instance");
  const RollNsView* const roll = reinterpret_cast<const RollNsView*>(&words_map);
  static_assert(!kRoll || (kDrain && !kSet), "the rollout instance is a drain instance of its own");
  const RollWaveNsView* const rwave = reinterpret_cast<const RollWaveNsView*>(&words_map);
  static_assert(!kWave || kRoll, "the rollout wave instance is a rollout instance");
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5, n_warps = blockDim.x >> 5;
  const uint32_t* words = table_bytes ? s_words : a.g_words;
  const uint32_t* order = table_bytes ? s_order : a.node_order;

  if (tid == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(s_mbar)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  // (no early griddepcontrol.launch_dependents: a dependent would only park its CTAs on SMs the
  // concurrent sweep wants; it still launches ahead and starts the moment this grid ends)
  pdl_wait_prior();  // the condense kernel's tables (and the request table a tick's scatter patched)
  if (tid == 0) {
    // TMA: the capacity vector and the domain index — and, scan form, the node-word table (a 2D
    // tensor of 256-word rows) and the node order — land in shared memory while the other threads
    // clear the holder table and take the pinned claims; one mbarrier collects the bytes
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(s_mbar)),
                 "r"(2u * table_bytes + free_bytes + first_bytes)
                 : "memory");
    if (table_bytes) {
      if (a.use_tensor_map) {
        asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
                         smem_u32(s_words)),
                     "l"(&words_map), "r"(smem_u32(s_mbar)), "r"(0), "r"(0)
                     : "memory");
      } else {
        bulk_load(s_words, a.g_words, table_bytes, s_mbar);
      }
      bulk_load(s_order, a.node_order, table_bytes, s_mbar);
    }
    bulk_load(s_free, a.g_dom_free, free_bytes, s_mbar);
    bulk_load(s_first, a.dom_first, first_bytes, s_mbar);
  }
  bool staged = false;
  uint32_t n_iter = 0, slice = 0;  // (kDrain; the other instances bound the loop by the parameter itself)
  if constexpr (kDrain) {
    n_iter = min(__ldcg(drain->n_items), drain->item_capacity);  // (an item the set refused is not in the list)
    slice = blockIdx.x * drain->slice_rows;
    mbar_wait(s_mbar);  // the overlays below write the staged capacities
    staged = true;
  }

  for (uint32_t it = blockIdx.x; it < (kDrain ? n_iter : a.n_namespaces); it += gridDim.x) {
    uint32_t ns = it, key = LWSE_NONE;
    if constexpr (kDrain) {
      const uint2 w = __ldcg(drain->items + it);
      key = w.x;
      ns = w.y;
    }
    uint4 ent = make_uint4(0u, 0u, 0u, 0u);  // kRoll: the entry's {first extra row, |E_i|, group range}
    uint4 wd = make_uint4(0u, 0u, 0u, 0u);   // kWave: the slot's {k, first list entry, list length, column rows}
    if constexpr (kWave) {
      wd = __ldcg(rwave->desc + key);
      ent = __ldcg(roll->ent + wd.x);
      ent.y += wd.w;  // the positions: the column's rows, then E_k's
    } else if constexpr (kRoll) {
      ent = __ldcg(roll->ent + key);
    }
    const uint32_t first = __ldcg(a.ns_first + ns), last_res = __ldcg(a.ns_first + ns + 1u), last = last_res + ent.y;
    if (tid == 0) {
      s_n_unp = 0u;
      s_n_cand = 0u;
      s_unsettled[0] = s_unsettled[1] = s_unsettled[2] = 0u;
    }
    for (uint32_t d = tid; d < a.n_domains; d += blockDim.x) s_hold[d] = ~0ull;
    __syncthreads();
    if (first >= last) continue;  // CTA-uniform
    // where results and the unpinned list go: the row (by position in this CTA's slice for kDrain)
    lwse_place_out* const obase = kDrain ? a.out + slice : a.out;
    const uint32_t ubase = kDrain ? slice : first;
    uint32_t skip_node = LWSE_NONE, od = LWSE_NONE, of = 0;  // kDrain: the drained node / domain, its staged capacity
    unsigned long long skip_bit = 0ull;                      // kSet: the column's bit in key_wave
    if constexpr (kSet) {
      const DrainNsView& dv = set->d;
      const uint32_t k = __ldcg(set->state), c = key;
      skip_bit = 1ull << c;
      for (uint32_t p = tid; p < last - first; p += blockDim.x)
        dv.marks[slice + p] = (__ldcg(set->u_wave + __ldcg(a.ns_rows + first + p)) & skip_bit) ? 1u : 0u;
      __syncthreads();
      for (uint32_t j = __ldcg(dv.u_first + k) + tid, end = __ldcg(dv.u_first + k + 1u); j < end; j += blockDim.x) {
        const uint32_t p = __ldcg(dv.pos + __ldcg(dv.u_rows + j));
        if (p >= first && p < last) dv.marks[slice + p - first] = 1u;
      }
      uint32_t kd = LWSE_NONE, kf = 0;
      if (dv.by_domain) {
        kd = k < a.n_domains ? k : LWSE_NONE;
      } else if (k < a.n_nodes) {
        skip_node = k;
        const uint4 nr = ldg_keep(reinterpret_cast<const uint4*>(a.nodes + k));
        const uint32_t fl = nr.w >> 16;
        if ((fl & LWSE_NODE_SCHEDULABLE) && (fl & LWSE_NODE_HAS_TOPOLOGY) && nr.z < a.n_domains) {
          const uint32_t cap = nr.w & 0xFFFFu, occ = occupancy_sum(a, a.occupancy, k);
          kf = cap > occ ? cap - occ : 0u;
          kd = nr.z;
        }
      }
      for (uint32_t d = tid; d < a.n_domains; d += blockDim.x) {
        uint32_t f = __ldcg(a.g_dom_free + d);
        if (dv.by_domain) {
          if (d == kd || (__ldcg(set->key_wave + d) & skip_bit)) f = 0u;
        } else {
          f -= __ldcg(set->drained + (size_t)c * a.n_domains + d) + (d == kd ? kf : 0u);
        }
        s_free[d] = f;
      }
      __syncthreads();
    } else if constexpr (kDrain && !kRoll) {
      const DrainNsView& dv = *drain;
      for (uint32_t p = tid; p < last - first; p += blockDim.x) dv.marks[slice + p] = 0u;
      __syncthreads();
      for (uint32_t j = __ldcg(dv.u_first + key) + tid, end = __ldcg(dv.u_first + key + 1u); j < end; j += blockDim.x) {
        const uint32_t p = __ldcg(dv.pos + __ldcg(dv.u_rows + j));
        if (p >= first && p < last) dv.marks[slice + p - first] = 1u;  // (LWSE_NONE: no namespace)
      }
      uint32_t lowered = 0;
      if (dv.by_domain) {
        od = key < a.n_domains ? key : LWSE_NONE;
      } else if (key < a.n_nodes) {
        const uint4 nr = ldg_keep(reinterpret_cast<const uint4*>(a.nodes + key));
        const uint32_t fl = nr.w >> 16;
        if ((fl & LWSE_NODE_SCHEDULABLE) && (fl & LWSE_NODE_HAS_TOPOLOGY) && nr.z < a.n_domains) {
          const uint32_t cap = nr.w & 0xFFFFu, occ = occupancy_sum(a, a.occupancy, key);
          lowered = cap > occ ? cap - occ : 0u;
          od = nr.z;
          skip_node = key;
        }
      }
      if (od != LWSE_NONE) {
        of = s_free[od];
        __syncthreads();  // every thread has read the staged value before thread 0 lowers it
        if (tid == 0) s_free[od] = dv.by_domain ? 0u : of - lowered;
      }
      __syncthreads();
    }
    auto req_at = [&](uint32_t r, uint32_t p) -> const uint4* {  // the request row at position p (row r)
      if constexpr (kWave) {
        if (p >= last_res) {
          const uint32_t q = p - last_res;
          if (q >= wd.w) return reinterpret_cast<const uint4*>(roll->extra + ent.x + (q - wd.w));
          uint32_t lo = wd.y, hi = wd.y + wd.z;  // the listed entry holding q: the last offset <= q
          while (hi - lo > 1u) {
            const uint32_t mid = (lo + hi) >> 1;
            if (__ldg(&rwave->col[mid].y) <= q) lo = mid; else hi = mid;
          }
          const uint4 c = __ldg(rwave->col + lo);
          return reinterpret_cast<const uint4*>(roll->extra + c.x + (q - c.y));
        }
      }
      if constexpr (kRoll) {
        if (p >= last_res) return reinterpret_cast<const uint4*>(roll->extra + ent.x + (p - last_res));
      }
      return reinterpret_cast<const uint4*>(a.reqs + r);
    };
    auto req_hi = [&](uint32_t r, uint32_t p) -> uint4 {  // the request's second half, U_k unpinned for kDrain
      uint4 hi = ldg_keep(req_at(r, p) + 1);
      if constexpr (kDrain && !kRoll) {
        if (__ldcg(drain->marks + slice + (p - first))) hi.w = LWSE_NONE;
      }
      return hi;
    };

    // ---- phase 1: pinned claims, the list of live unpinned requests ----
    // the first kNsKeep requests of a thread stay in registers until their result is written
    uint4 k_lo[kNsKeep], k_hi[kNsKeep];
    uint32_t k_dom[kNsKeep], k_row[kNsKeep];
    auto row_of = [&](uint32_t p) -> uint32_t {  // position in the namespace's range -> request row
      if constexpr (kRoll) {
        if (p >= last_res) return roll->n_resident + (p - last_res);
      }
      if constexpr (kIndexed) return __ldcg(a.ns_rows + p);
      return p;
    };
#pragma unroll
    for (uint32_t j = 0; j < kNsKeep; j++) {  // all request loads of the thread in flight together
      const uint32_t p = first + tid + j * blockDim.x;
      if (p < last) {
        const uint32_t r = row_of(p);
        if constexpr (kIndexed) k_row[j] = r;
        k_lo[j] = ldg_keep(req_at(r, p));
        k_hi[j] = req_hi(r, p);
      }
    }
    // x: where the request's result and list entry go — its row, or (kDrain) its position in the namespace
    auto claim = [&](uint32_t r, uint32_t x, const uint4 lo, const uint4 hi) -> uint32_t {
      const uint32_t leader = hi.w;
      uint32_t d = LWSE_NONE;
      if (leader == LWSE_NONE) {
        const bool dead = (int32_t)hi.z < 1;
        const uint4 row = make_uint4(LWSE_NONE, LWSE_NONE, dead ? LWSE_PLACE_UNSCHEDULABLE : 0u, 0u);
        *reinterpret_cast<uint4*>(obase + x) = row;
        if (dead) {
          diff_row(a, r, row);
        } else {
          const uint32_t k = atomicAdd(&s_n_unp, 1u);
          a.unpinned[ubase + k] = x;
          if (k < kNsCache) {
            NsReq q;
            q.key = ns_place_key(u64_of(lo.x, lo.y), r, false);
            q.r = x;
            q.key_lo = lo.z;
            q.key_hi = lo.w;
            q.size = hi.z;
            q.cur = LWSE_NONE;
            q.dead = 0u;
            s_req[k] = q;
          }
        }
      } else {
        if (leader < a.n_nodes) {
          const uint4 nr = ldg_keep(reinterpret_cast<const uint4*>(a.nodes + leader));
          if (((nr.w >> 16) & LWSE_NODE_HAS_TOPOLOGY) && nr.z < a.n_domains) d = nr.z;
        }
        if (d != LWSE_NONE) atomicMin(s_hold + d, ns_place_key(u64_of(lo.x, lo.y), r, true));
      }
      return d;
    };
    auto result = [&](uint32_t r, uint32_t x, const uint4 lo, const uint4 hi, uint32_t d) {
      if (hi.w == LWSE_NONE) return;
      uint32_t flags = LWSE_PLACE_PINNED;
      if (d != LWSE_NONE) flags |= s_hold[d] == ns_place_key(u64_of(lo.x, lo.y), r, true) ? LWSE_PLACE_PLACED : LWSE_PLACE_CONFLICT;
      const uint4 row = make_uint4(d, hi.w, flags, 0u);
      *reinterpret_cast<uint4*>(obase + x) = row;
      diff_row(a, r, row);
    };
#pragma unroll
    for (uint32_t j = 0; j < kNsKeep; j++) {
      const uint32_t p = first + tid + j * blockDim.x;
      if (p < last) {
        const uint32_t r = kIndexed ? k_row[j] : p;
        k_dom[j] = claim(r, kDrain ? p - first : r, k_lo[j], k_hi[j]);
      }
    }
    for (uint32_t p = first + tid + kNsKeep * blockDim.x; p < last; p += blockDim.x) {  // big namespaces: the rest, unkept
      const uint32_t r = row_of(p);
      claim(r, kDrain ? p - first : r, ldg_keep(req_at(r, p)), req_hi(r, p));
    }
    __syncthreads();
    // results of the pinned requests: final from here on (pinned keys are below every unpinned key)
#pragma unroll
    for (uint32_t j = 0; j < kNsKeep; j++) {
      const uint32_t p = first + tid + j * blockDim.x;
      if (p < last) {
        const uint32_t r = kIndexed ? k_row[j] : p;
        result(r, kDrain ? p - first : r, k_lo[j], k_hi[j], k_dom[j]);
      }
    }
    for (uint32_t p = first + tid + kNsKeep * blockDim.x; p < last; p += blockDim.x) {
      const uint32_t r = row_of(p);
      const uint4 lo = ldg_keep(req_at(r, p)), hi = req_hi(r, p);
      uint32_t d = LWSE_NONE;
      if (hi.w != LWSE_NONE && hi.w < a.n_nodes) {
        const uint4 nr = ldg_keep(reinterpret_cast<const uint4*>(a.nodes + hi.w));
        if (((nr.w >> 16) & LWSE_NODE_HAS_TOPOLOGY) && nr.z < a.n_domains) d = nr.z;
      }
      result(r, kDrain ? p - first : r, lo, hi, d);
    }
    const uint32_t n_unp = s_n_unp;
    if (n_unp == 0u && !kDrain) {  // (kDrain: the diff below still runs; the rounds end at once)
      __syncthreads();
      continue;
    }
    if (tid == 0) atomicAdd(a.counters + 1, n_unp);
    if (!staged) {  // the first namespace with work waits for the staged tables
      mbar_wait(s_mbar);
      staged = true;
    }
    uint32_t n_cand = 0;
    if constexpr (!kScan) {
      // The domains an unpinned request can ever win: no pinned holder (a pinned key is below every
      // unpinned key) and capacity left.  The rounds look at this list only; the holder table of
      // the unpinned claims is indexed by the list position.
      for (uint32_t d = tid; d < a.n_domains; d += blockDim.x) {
        const uint32_t fr = s_free[d];
        if (s_hold[d] == ~0ull && fr != 0u) {
          const uint32_t c = atomicAdd(&s_n_cand, 1u);
          s_cand[c] = make_uint2(d, fr);
          s_holdc[c] = ~0ull;
          s_slot[d] = c;
        }
      }
      __syncthreads();
      n_cand = s_n_cand;
    }

    // ---- deferred-acceptance rounds of this namespace, one warp per request ----
    uint32_t round = 0;
    for (;; round++) {
      // three rotating counters: the one for round k+1 is cleared during round k, when nobody can
      // still be reading it (it was last read after round k-2)
      uint32_t* unsettled_ctr = &s_unsettled[round % 3u];
      if (tid == 0) s_unsettled[(round + 1u) % 3u] = 0u;
      uint32_t scans = 0;
      for (uint32_t k = warp; k < n_unp; k += n_warps) {
        NsReq q;
        const bool cached = k < kNsCache;
        if (cached) {
          q = s_req[k];
        } else {  // overflow: the state lives in the result row (written by this warp only)
          q.r = __ldcg(a.unpinned + ubase + k);
          const uint32_t qrow = kRoll ? row_of(first + q.r) : kDrain ? __ldcg(a.ns_rows + first + q.r) : q.r;
          const uint4 o = __ldcg(reinterpret_cast<const uint4*>(obase + q.r));
          const uint4* const qreq = kRoll ? req_at(qrow, first + q.r) : reinterpret_cast<const uint4*>(a.reqs + qrow);
          const uint4 lo = ldg_keep(qreq), hi = ldg_keep(qreq + 1);
          q.key = ns_place_key(u64_of(lo.x, lo.y), qrow, false);
          q.key_lo = lo.z;
          q.key_hi = lo.w;
          q.size = hi.z;
          q.cur = o.x;
          if (!kScan && o.x != LWSE_NONE) q.cur = s_slot[o.x];
          q.dead = (o.z & LWSE_PLACE_UNSCHEDULABLE) ? 1u : 0u;
        }
        __syncwarp();  // every lane has its copy before lane 0 updates the cache entry below
        if (q.dead) continue;  // warp-uniform
        const unsigned long long key = q.key;
        const uint32_t key_lo = q.key_lo, key_hi = q.key_hi, size = q.size, r = q.r;
        if (q.cur != LWSE_NONE && (kScan ? s_hold[q.cur] : s_holdc[q.cur]) == key) continue;  // still holds what it proposed to
        scans++;
        uint32_t H = 0, best_d = LWSE_NONE, best_n = LWSE_NONE, best_c = LWSE_NONE;
        if constexpr (!kScan) {
          // Level 1 — the domain, over the candidate list in shared memory (holders change under
          // our feet during a round; a stale reading can only make a proposal fail: holder keys
          // only decrease).
          uint32_t my_hi = 0, my_d = LWSE_NONE, my_c = LWSE_NONE;
#pragma unroll 4
          for (uint32_t c = lane; c < n_cand; c += 32u) {
            const uint2 cd = s_cand[c];
            const unsigned long long hk = s_holdc[c];
            const uint32_t h = (cd.y >= size && hk >= key) ? (mix32n(key_lo ^ (cd.x * 0x9E3779B1u)) | 1u) : 0u;
            if (h > my_hi || (h == my_hi && h != 0u && cd.x < my_d)) {  // ties keep the lower domain
              my_hi = h;
              my_d = cd.x;
              my_c = c;
            }
          }
          H = __reduce_max_sync(0xFFFFFFFFu, my_hi);
          if (H != 0u) {
            best_d = __reduce_min_sync(0xFFFFFFFFu, my_hi == H ? my_d : LWSE_NONE);
            const uint32_t owner = __ffs(__ballot_sync(0xFFFFFFFFu, my_hi == H && my_d == best_d)) - 1u;
            best_c = __shfl_sync(0xFFFFFFFFu, my_c, (int)owner);
            // Level 2 — the node: the domain's run of the condensed (free | node) words.
            const uint32_t f2 = s_first[best_d], l2 = s_first[best_d + 1u];
            uint32_t my_lo = 0, my_n = LWSE_NONE;
            for (uint32_t i = f2 + lane; i < l2; i += 32u) {
              const uint32_t w = __ldcg(a.g_nodes2 + i);
              if ((w >> 28) == 0u) continue;
              const uint32_t n = w & 0x0FFFFFFFu;
              if constexpr (kSet) {
                if (n == skip_node || (!set->d.by_domain && (__ldcg(set->key_wave + n) & skip_bit))) continue;  // cordoned
              } else if constexpr (kDrain) {
                if (n == skip_node) continue;  // cordoned
              }
              const uint32_t l = ((w >> 28) << 28) | (mix32n(key_hi ^ (n * 0x85EBCA77u)) >> 4);
              if (l > my_lo || (l == my_lo && n < my_n)) {
                my_lo = l;
                my_n = n;
              }
            }
            const uint32_t L = __reduce_max_sync(0xFFFFFFFFu, my_lo);
            best_n = __reduce_min_sync(0xFFFFFFFFu, (my_lo == L && L != 0u) ? my_n : LWSE_NONE);
          }
        } else {
          // Brute force: every (request, node) pair of the staged table.  Lexicographic arg-max of
          // (domain score, lower domain, node score, lower node) — the two-level result.
          // (the usable-node count from the staged index, not a launch parameter: a replayed tick graph
          // keeps its parameters while node-row patches change the count)
          uint32_t my_hi = 0, my_d = LWSE_NONE, my_lo = 0, my_n = LWSE_NONE;
          const uint32_t n_usable = s_first[a.n_domains];
          for (uint32_t i = lane; i < n_usable; i += 32u) {
            const uint32_t w = words[i], d = w & 0x0FFFFFFFu;
            if ((w >> 28) == 0u || s_free[d] < size || s_hold[d] < key) continue;
            const uint32_t h = mix32n(key_lo ^ (d * 0x9E3779B1u)) | 1u;
            if (h < my_hi || (h == my_hi && d > my_d)) continue;
            const uint32_t n = order[i];
            const uint32_t l = ((w >> 28) << 28) | (mix32n(key_hi ^ (n * 0x85EBCA77u)) >> 4);
            const bool better = h > my_hi || d < my_d || l > my_lo || (l == my_lo && n < my_n);
            if (better) {
              my_hi = h;
              my_d = d;
              my_lo = l;
              my_n = n;
            }
          }
          H = __reduce_max_sync(0xFFFFFFFFu, my_hi);
          if (H != 0u) {
            best_d = __reduce_min_sync(0xFFFFFFFFu, my_hi == H ? my_d : LWSE_NONE);
            const bool in = my_hi == H && my_d == best_d;
            const uint32_t L = __reduce_max_sync(0xFFFFFFFFu, in ? my_lo : 0u);
            best_n = __reduce_min_sync(0xFFFFFFFFu, (in && my_lo == L && L != 0u) ? my_n : LWSE_NONE);
          }
          best_c = best_d;
        }
        if (lane == 0) {
          if (H == 0u || best_n == LWSE_NONE) {  // nothing feasible now, and the feasible set only shrinks
            store_row(obase + r, LWSE_NONE, LWSE_NONE, LWSE_PLACE_UNSCHEDULABLE, 0u);
            if (cached) s_req[k].dead = 1u;
          } else {
            store_row(obase + r, best_d, best_n, LWSE_PLACE_PLACED, H);
            if (cached) s_req[k].cur = best_c;
            // A claim on an empty domain settles at once; any other outcome leaves somebody without
            // a domain who proposes again next round: count it.
            const unsigned long long old = atomicMin((kScan ? s_hold : s_holdc) + best_c, key);
            if (old != ~0ull) atomicAdd(unsettled_ctr, 1u);
          }
        }
        __syncwarp();
      }
      if (lane == 0 && scans) atomicAdd(a.counters + 3, scans);
      __syncthreads();
      const uint32_t unsettled = *unsettled_ctr;
      if (unsettled == 0u || round > n_unp + 2u) break;
    }
    if (tid == 0) atomicMax(a.counters + 0, round + 1u);
    // a tick's change list: the rows of the unpinned requests are final now
    if (a.prev != nullptr) {
      for (uint32_t k = tid; k < n_unp; k += blockDim.x) {
        const uint32_t r = k < kNsCache ? s_req[k].r : __ldcg(a.unpinned + first + k);
        diff_row(a, r, __ldcg(reinterpret_cast<const uint4*>(a.out + r)));
      }
    }
    __syncthreads();
    if constexpr (kRoll) {  // the namespace's rows against the baseline, E_i's rows, reduced in the CTA
      const DrainNsView& dv = roll->d;
      uint32_t c[kRollCounts] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
      for (uint32_t p = first + tid; p < last; p += blockDim.x) {
        const uint4 v = __ldcg(reinterpret_cast<const uint4*>(obase + (p - first)));
        const bool is = (v.z & LWSE_PLACE_PLACED) != 0u;
        c[8] += is ? 1u : 0u;
        c[9] += (v.z & LWSE_PLACE_UNSCHEDULABLE) ? 1u : 0u;
        c[10] += (v.z & LWSE_PLACE_CONFLICT) ? 1u : 0u;
        if (p >= last_res) {  // a row of E_i
          c[0] += is ? 1u : 0u;
          c[1] += is ? 0u : 1u;
          continue;
        }
        const uint32_t r = row_of(p);
        const uint4 o = __ldg(reinterpret_cast<const uint4*>(dv.base + r));
        const bool was = (o.z & LWSE_PLACE_PLACED) != 0u;
        const uint32_t grp = __ldg(&a.reqs[r].group);
        bool own = grp - ent.z < ent.w;
        if constexpr (kWave) {  // a lost row: the listed entries' ranges too
          for (uint32_t j = wd.y; !own && was && !is && j < wd.y + wd.z; j++) {
            const uint4 c = __ldg(rwave->col + j);
            own = grp - c.z < c.w;
          }
        }
        c[2] += (own && was && !is) ? 1u : 0u;
        c[3] += (!own && was && !is) ? 1u : 0u;
        c[4] += (v.x != o.x || v.y != o.y || v.z != o.z || v.w != o.w) ? 1u : 0u;
        c[5] += (was && !is) ? 1u : 0u;
        c[6] += (was && is && o.x != v.x) ? 1u : 0u;
        c[7] += (!was && is) ? 1u : 0u;
        c[8] -= was ? 1u : 0u;
        c[9] -= (o.z & LWSE_PLACE_UNSCHEDULABLE) ? 1u : 0u;
        c[10] -= (o.z & LWSE_PLACE_CONFLICT) ? 1u : 0u;
      }
      uint32_t* const s_rcnt = reinterpret_cast<uint32_t*>(s_req);  // (the request cache is free after the rounds)
      if (tid < kRollCounts) s_rcnt[tid] = 0u;
      __syncthreads();
#pragma unroll
      for (uint32_t f = 0; f < kRollCounts; f++) {
        const uint32_t sum = __reduce_add_sync(0xFFFFFFFFu, c[f]);
        if (lane == 0 && sum) atomicAdd(&s_rcnt[f], sum);
      }
      __syncthreads();
      uint32_t* erow = dv.rows + (size_t)key * 16u;
      if (tid < kRollCounts && s_rcnt[tid]) atomicAdd(erow + 4u + tid, s_rcnt[tid]);
      if (tid == kRollCounts) atomicAdd(erow + 15u, 1u);  // namespaces_solved
      __syncthreads();
    } else if constexpr (kDrain) {  // the namespace's rows against the baseline, reduced in the CTA, one atomic per field
      const DrainNsView& dv = *drain;
      uint32_t c[kDrainCounts] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
      for (uint32_t p = first + tid; p < last; p += blockDim.x) {
        const uint4 v = __ldcg(reinterpret_cast<const uint4*>(obase + (p - first)));
        const uint4 o = __ldg(reinterpret_cast<const uint4*>(dv.base + row_of(p)));
        drain_place_count(c, o, v, __ldcg(dv.marks + slice + (p - first)) != 0u);
      }
      uint32_t* const s_dcnt = reinterpret_cast<uint32_t*>(s_req);  // (the request cache is free after the rounds)
      if (tid < kDrainCounts) s_dcnt[tid] = 0u;
      __syncthreads();
#pragma unroll
      for (uint32_t f = 0; f < kDrainCounts; f++) {
        const uint32_t sum = __reduce_add_sync(0xFFFFFFFFu, c[f]);
        if (lane == 0 && sum) atomicAdd(&s_dcnt[f], sum);
      }
      __syncthreads();
      uint32_t* krow = dv.rows + (size_t)key * 16u;
      if (tid < kDrainCounts && s_dcnt[tid]) atomicAdd(krow + 2u + tid, s_dcnt[tid]);
      if (tid == kDrainCounts) atomicAdd(krow + 11u, 1u);  // namespaces_solved
      if (tid == 0 && od != LWSE_NONE) s_free[od] = of;
      __syncthreads();
    }
  }
  if (!staged) mbar_wait(s_mbar);  // never leave a bulk copy in flight behind a CTA that exits
}

// --------------------------------------------------------------------------
// launcher
// --------------------------------------------------------------------------
static size_t up256(size_t v) { return (v + 255) / 256 * 256; }

// scratch: [words (rows x 1 KB)] [nodes2 (same)] [dom_free] [ns_first] [unpinned] [counters: 2 blocks of 8 words]
//          [indexed form: ns_rows] [ns_count] [ns_cursor]
struct NsLayout {
  size_t words, nodes2, dom_free, ns_first, unpinned, counters, ns_rows, ns_count, ns_cursor, total;
  uint32_t word_rows;
};
static NsLayout ns_layout(uint32_t n_nodes, uint32_t n_domains, uint32_t n_reqs, uint32_t n_namespaces) {
  NsLayout l{};
  l.word_rows = (n_nodes + 255u) / 256u;
  if (l.word_rows == 0) l.word_rows = 1;
  size_t off = 0;
  l.words = off;
  off += up256((size_t)l.word_rows * 1024);
  l.nodes2 = off;
  off += up256((size_t)l.word_rows * 1024);
  l.dom_free = off;
  off += up256((size_t)n_domains * 4 + 16);
  l.ns_first = off;
  off += up256(((size_t)n_namespaces + 2) * 4);
  l.unpinned = off;
  off += up256((size_t)n_reqs * 4 + 16);
  l.counters = off;
  off += 256;
  l.ns_rows = off;
  off += up256((size_t)n_reqs * 4 + 16);
  l.ns_count = off;
  off += up256((size_t)n_namespaces * 4 + 16);
  l.ns_cursor = off;
  off += up256((size_t)n_namespaces * 4 + 16);
  l.total = off;
  return l;
}
size_t place_ns_scratch_bytes(uint32_t n_nodes, uint32_t n_domains, uint32_t n_reqs, uint32_t n_namespaces) {
  return ns_layout(n_nodes, n_domains, n_reqs, n_namespaces).total;
}

// shared memory of the namespace kernel: the scan form with / without the staged word table, the
// two-level form (candidate list, holder table by candidate, slot of domain)
static size_t ns_smem_bytes(uint32_t word_rows, uint32_t n_domains, bool scan, bool stage) {
  const size_t free_bytes = ((size_t)n_domains * 4 + 15) & ~(size_t)15;
  const size_t base = free_bytes + ((((size_t)n_domains + 1) * 4 + 15) & ~(size_t)15) + (size_t)n_domains * 8 + 256 * 32 + 16 + 128;
  if (scan) return base + (stage ? (size_t)word_rows * 2048 : 0);
  return base + (size_t)n_domains * 16 + free_bytes;
}
bool place_ns_supported(uint32_t n_nodes, uint32_t n_domains) {
  return ns_smem_bytes((n_nodes + 255u) / 256u, n_domains, false, false) <= 200u * 1024u && n_domains < (1u << 28) &&
         n_nodes < (1u << 28);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static bool encode_words_map(CUtensorMap* map, void* g_words, uint32_t word_rows) {
  static EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
      p = nullptr;
    (void)cudaGetLastError();
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  if (!fn || word_rows == 0 || word_rows > 256) return false;
  const cuuint64_t dims[2] = {256, word_rows};
  const cuuint64_t strides[1] = {1024};
  const cuuint32_t box[2] = {256, word_rows};
  const cuuint32_t estr[2] = {1, 1};
  return fn(map, CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, g_words, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Returns kernels launched or -1.  `fresh`: the scratch was (re)allocated: zero it first.
int launch_place_ns(const lwse_node_rec* d_nodes, const uint32_t* d_dom_first, const uint32_t* d_node_order, uint32_t n_nodes,
                    uint32_t n_domains, const lwse_place_req* d_reqs, uint32_t n_reqs,
                    const uint32_t* d_occupancy, uint32_t n_parts, uint64_t part_stride_bytes, uint32_t n_namespaces,
                    lwse_place_out* d_out, void* d_scratch, size_t scratch_bytes, bool fresh, uint32_t call_index, bool scan,
                    int sm_count, cudaStream_t s, const uint32_t** d_counters_out, bool first_pdl,
                    const PlaceNsChanges* changes, const PlaceNsExchange* xch, PlaceNsIndex index) {
  const NsLayout l = ns_layout(n_nodes, n_domains, n_reqs, n_namespaces);
  if (scratch_bytes < l.total || n_reqs > 0xFFFFFFu) return -(int)cudaErrorInvalidValue;
  uint8_t* base = static_cast<uint8_t*>(d_scratch);
  cudaError_t e = cudaSuccess;
  if (fresh) {
    e = cudaMemsetAsync(base, 0, l.total, s);
    if (e != cudaSuccess) return -(int)e;
  }
  PlaceNsArgs a{};
  a.nodes = d_nodes;
  a.reqs = d_reqs;
  a.occupancy = d_occupancy;
  a.out = d_out;
  a.dom_first = d_dom_first;
  a.node_order = d_node_order;
  a.g_words = reinterpret_cast<uint32_t*>(base + l.words);
  a.g_nodes2 = reinterpret_cast<uint32_t*>(base + l.nodes2);
  a.g_dom_free = reinterpret_cast<uint32_t*>(base + l.dom_free);
  a.ns_first = reinterpret_cast<uint32_t*>(base + l.ns_first);
  a.unpinned = reinterpret_cast<uint32_t*>(base + l.unpinned);
  if (index != kNsIndexNone) {
    if (fresh) index = kNsIndexBuild;  // (the zeroed scratch holds no index)
    a.ns_rows = reinterpret_cast<uint32_t*>(base + l.ns_rows);
    a.ns_count = reinterpret_cast<uint32_t*>(base + l.ns_count);
    a.ns_cursor = reinterpret_cast<uint32_t*>(base + l.ns_cursor);
  }
  // counters: 256 bytes = 8 blocks of 8 words.  Blocks 0 / 1 alternate between calls (a call clears the
  // block the next one uses); blocks 2 / 3 belong to the tick slots.
  const int tick_slot = (changes && changes->prev) ? changes->tick_slot : -1;
  if (tick_slot >= 0) {
    a.counters = reinterpret_cast<uint32_t*>(base + l.counters) + (2u + (uint32_t)(tick_slot & 1)) * 8u;
    a.next_counters = nullptr;
  } else {
    a.counters = reinterpret_cast<uint32_t*>(base + l.counters) + (call_index & 1u) * 8u;
    a.next_counters = reinterpret_cast<uint32_t*>(base + l.counters) + ((call_index + 1u) & 1u) * 8u;
  }
  a.n_nodes = n_nodes;
  a.n_domains = n_domains;
  a.n_reqs = n_reqs;
  a.n_namespaces = n_namespaces;
  a.n_parts = d_occupancy ? (n_parts ? n_parts : 1u) : 0u;
  a.part_stride_bytes = part_stride_bytes;
  a.word_rows = l.word_rows;
  a.scan = scan ? 1u : 0u;
  if (xch && xch->step_ctr) {
    a.xch_step = xch->step_ctr;
    a.xch_half_bytes = xch->half_bytes;
    a.xch_lagged = xch->lagged ? 1u : 0u;
  }
  if (d_counters_out) *d_counters_out = a.counters;
  if (changes && changes->prev) {
    a.prev = changes->prev;
    a.chg_rows = changes->rows;
    a.chg_outs = changes->outs;
    a.chg_count = changes->count;
    a.chg_capacity = changes->capacity;
  }

  // does the word table fit next to the holder table?  (227 KB of shared memory per CTA)
  const size_t with_words = ns_smem_bytes(l.word_rows, n_domains, true, true);
  a.stage_words = (scan && with_words <= 100u * 1024u) ? 1u : 0u;  // two CTAs per SM keep their tables side by side
  const size_t smem = ns_smem_bytes(l.word_rows, n_domains, scan, a.stage_words != 0);
  // the tensor map of the word table: re-encoded when the scratch moved
  static thread_local CUtensorMap map;
  static thread_local void* map_for = nullptr;
  static thread_local uint32_t map_rows = 0;
  static thread_local bool map_ok = false;
  if (a.stage_words && (map_for != a.g_words || map_rows != l.word_rows)) {
    map_ok = encode_words_map(&map, a.g_words, l.word_rows);
    map_for = a.g_words;
    map_rows = l.word_rows;
  }
  a.use_tensor_map = (a.stage_words && map_ok) ? 1u : 0u;

  int launched = 2;
  // first_pdl: the predecessor on the stream is a kernel — programmatically dependent then (every
  // kernel here waits at its top, before its first read, so this is safe even behind a tick's scatter
  // kernel, whose tail the launch latency overlaps); behind a copy / memset / event an ordinary launch
  bool pdl = first_pdl;
  if (index == kNsIndexBuild) {  // count -> scan -> fill, a thread per request
    uint64_t grid = ((uint64_t)n_reqs + 255) / 256;
    if (grid < 1) grid = 1;
    if (grid > (uint64_t)sm_count * 8u) grid = (uint64_t)sm_count * 8u;
    e = launch_pdl(place_index_count_kernel, dim3((unsigned)grid), dim3(256), 0, s, pdl, a);
    if (e == cudaSuccess)
      e = launch_pdl(place_index_scan_kernel, dim3(1), dim3(kIndexScanThreads), 0, s, true,
                     IndexScanArgs{a.ns_count, a.ns_first, a.ns_cursor, n_namespaces});
    if (e == cudaSuccess) e = launch_pdl(place_index_fill_kernel, dim3((unsigned)grid), dim3(256), 0, s, true, a);
    if (e != cudaSuccess) return -(int)e;
    pdl = true;
    launched += 3;
  }
  {  // condense: a warp per domain, a thread per request
    uint64_t threads = (uint64_t)n_domains * 32u;
    if (threads < n_reqs) threads = n_reqs;
    uint64_t grid = (threads + 255) / 256;
    if (grid < 1) grid = 1;
    if (grid > (uint64_t)sm_count * 8u) grid = (uint64_t)sm_count * 8u;
    e = launch_pdl(place_condense_kernel, dim3((unsigned)grid), dim3(256), 0, s, pdl, a);
    if (e != cudaSuccess) return -(int)e;
    if (changes && changes->mid_event) {
      e = cudaEventRecord(static_cast<cudaEvent_t>(changes->mid_event), s);
      if (e != cudaSuccess) return -(int)e;
    }
  }
  {
    unsigned grid = n_namespaces < (unsigned)sm_count * 2u ? n_namespaces : (unsigned)sm_count * 2u;
    if (grid < 1u) grid = 1u;
    const bool indexed = index != kNsIndexNone;
    auto kern = scan ? (indexed ? place_ns_kernel<true, true> : place_ns_kernel<true, false>)
                     : (indexed ? place_ns_kernel<false, true> : place_ns_kernel<false, false>);
    const int variant = (scan ? 1 : 0) | (indexed ? 2 : 0);
    static thread_local size_t attr_set[4] = {0, 0, 0, 0};
    if (smem > attr_set[variant]) {
      e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (e != cudaSuccess) return -(int)e;
      attr_set[variant] = smem;
    }
    e = launch_pdl(kern, dim3(grid), dim3(scan ? kNsScanThreads : kNsThreads), smem, s, true, a, map);
    if (e != cudaSuccess) return -(int)e;
  }
  return launched;
}

// --------------------------------------------------------------------------
// what-if rounds (lwse_resident_place_whatif)
// --------------------------------------------------------------------------
// The what-if solves only the namespaces its patches touch: the namespace index it builds holds the
// rows of touched namespaces alone, so the namespace kernel's CTAs of the others see an empty range
// and its output keeps their rows (a copy of the baseline).  Exact, because namespaces share nothing
// but the capacity snapshot, which a what-if does not change.  The same count -> scan -> fill as the
// tick's index, with a mask: separate kernels, so that the tick's instances stay as they are.
struct WhatIfIndexArgs {
  const lwse_place_req* reqs;
  const uint8_t* touched;  // n_namespaces: 1 = solve this namespace
  uint32_t* ns_count;
  uint32_t* ns_cursor;
  uint32_t* ns_rows;
  uint32_t n_reqs, n_namespaces;
};

__device__ __forceinline__ uint32_t whatif_ns_of(const WhatIfIndexArgs& a, uint32_t i) {
  if (i >= a.n_reqs) return LWSE_NONE;
  const uint32_t v = __ldcg(reinterpret_cast<const uint32_t*>(a.reqs + i) + 5);  // .ns (rows the scatter just patched)
  return (v < a.n_namespaces && a.touched[v]) ? v : LWSE_NONE;
}

__global__ void __launch_bounds__(256) place_whatif_count_kernel(const WhatIfIndexArgs a) {
  const uint32_t lane = threadIdx.x & 31u, stride = gridDim.x * blockDim.x;
  for (uint32_t base = (blockIdx.x * blockDim.x + threadIdx.x) & ~31u; base < a.n_reqs; base += stride) {
    const uint32_t v = whatif_ns_of(a, base + lane);
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, v);
    if (v != LWSE_NONE && lane == (uint32_t)__ffs(peers) - 1u) atomicAdd(a.ns_count + v, (uint32_t)__popc(peers));
  }
}

__global__ void __launch_bounds__(256) place_whatif_fill_kernel(const WhatIfIndexArgs a) {
  const uint32_t lane = threadIdx.x & 31u, stride = gridDim.x * blockDim.x;
  for (uint32_t base = (blockIdx.x * blockDim.x + threadIdx.x) & ~31u; base < a.n_reqs; base += stride) {
    const uint32_t i = base + lane, v = whatif_ns_of(a, i);
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, v);
    const uint32_t leader = (uint32_t)__ffs(peers) - 1u;
    uint32_t pos = 0;
    if (v != LWSE_NONE && lane == leader) pos = atomicAdd(a.ns_cursor + v, (uint32_t)__popc(peers));
    pos = __shfl_sync(0xFFFFFFFFu, pos, (int)leader);
    if (v != LWSE_NONE) a.ns_rows[pos + (uint32_t)__popc(peers & ((1u << lane) - 1u))] = i;
  }
}

// The masked namespace index in the namespace-form scratch `d_scratch` (laid out as launch_place_ns
// lays it out for the same geometry; ns_count zero before, and again after).
int launch_place_whatif_index(const lwse_place_req* d_reqs, uint32_t n_reqs, uint32_t n_namespaces, const uint8_t* d_touched,
                              uint32_t n_nodes, uint32_t n_domains, void* d_scratch, int sm_count, cudaStream_t s) {
  const NsLayout l = ns_layout(n_nodes, n_domains, n_reqs, n_namespaces);
  uint8_t* base = static_cast<uint8_t*>(d_scratch);
  WhatIfIndexArgs a{};
  a.reqs = d_reqs;
  a.touched = d_touched;
  a.ns_count = reinterpret_cast<uint32_t*>(base + l.ns_count);
  a.ns_cursor = reinterpret_cast<uint32_t*>(base + l.ns_cursor);
  a.ns_rows = reinterpret_cast<uint32_t*>(base + l.ns_rows);
  a.n_reqs = n_reqs;
  a.n_namespaces = n_namespaces;
  uint64_t grid = ((uint64_t)n_reqs + 255) / 256;
  if (grid < 1) grid = 1;
  if (grid > (uint64_t)sm_count * 8u) grid = (uint64_t)sm_count * 8u;
  place_whatif_count_kernel<<<(unsigned)grid, 256, 0, s>>>(a);
  if (const int r = launch_result(0); r < 0) return r;
  place_index_scan_kernel<<<1, kIndexScanThreads, 0, s>>>(
      IndexScanArgs{a.ns_count, reinterpret_cast<uint32_t*>(base + l.ns_first), a.ns_cursor, n_namespaces});
  if (const int r = launch_result(0); r < 0) return r;
  place_whatif_fill_kernel<<<(unsigned)grid, 256, 0, s>>>(a);
  return launch_result(3);
}

// request row -> its position in the namespace index (rows of no namespace keep the caller's LWSE_NONE)
__global__ void __launch_bounds__(256) drain_place_pos_kernel(const uint32_t* ns_first, const uint32_t* ns_rows,
                                                              uint32_t n_namespaces, uint32_t* pos) {
  const uint32_t n = __ldcg(ns_first + n_namespaces);
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) pos[__ldcg(ns_rows + p)] = p;
}

// The drain-placement solve (lwse_resident_drain_place_cost): the capacities of the resident node index (the
// condense kernel's part A alone: n_reqs = 0 leaves the request rows and the index alone), then the drain
// instance over p->grid CTAs.  The round scratch holds the namespace index of every namespace
// (launch_place_whatif_index with every namespace touched).
int launch_place_ns_drain(const DrainPlaceLaunch* p, int sm_count, cudaStream_t s) {
  const NsLayout l = ns_layout(p->n_nodes, p->n_domains, p->n_reqs, p->n_namespaces);
  if (p->round_bytes < l.total || p->n_reqs > 0xFFFFFFu) return -(int)cudaErrorInvalidValue;
  uint8_t* base = static_cast<uint8_t*>(p->round);
  PlaceNsArgs a{};
  a.nodes = p->nodes;
  a.reqs = p->reqs;
  a.occupancy = p->occupancy;
  a.dom_first = p->dom_first;
  a.node_order = p->node_order;
  a.g_words = reinterpret_cast<uint32_t*>(base + l.words);
  a.g_nodes2 = reinterpret_cast<uint32_t*>(base + l.nodes2);
  a.g_dom_free = reinterpret_cast<uint32_t*>(base + l.dom_free);
  a.ns_first = reinterpret_cast<uint32_t*>(base + l.ns_first);
  a.ns_rows = reinterpret_cast<uint32_t*>(base + l.ns_rows);
  a.ns_count = reinterpret_cast<uint32_t*>(base + l.ns_count);
  a.ns_cursor = reinterpret_cast<uint32_t*>(base + l.ns_cursor);
  a.counters = reinterpret_cast<uint32_t*>(base + l.counters) + 4u * 8u;  // a block no other call uses
  a.n_nodes = p->n_nodes;
  a.n_domains = p->n_domains;
  a.n_namespaces = p->n_namespaces;
  a.n_parts = 1u;
  a.word_rows = l.word_rows;
  {
    uint64_t grid = ((uint64_t)p->n_domains * 32u + 255) / 256;
    if (grid < 1) grid = 1;
    if (grid > (uint64_t)sm_count * 8u) grid = (uint64_t)sm_count * 8u;
    place_condense_kernel<<<(unsigned)grid, 256, 0, s>>>(a);  // (a.n_reqs = 0: capacities only)
    grid = ((uint64_t)p->n_reqs + 255) / 256;
    if (grid < 1) grid = 1;
    if (grid > (uint64_t)sm_count * 8u) grid = (uint64_t)sm_count * 8u;
    drain_place_pos_kernel<<<(unsigned)grid, 256, 0, s>>>(a.ns_first, a.ns_rows, p->n_namespaces, p->pos);
    if (const int r = launch_result(0); r < 0) return r;
  }
  DrainNsView v{};
  v.items = p->items;
  v.n_items = p->counts + 4;
  v.item_capacity = p->item_capacity;
  v.u_first = p->u_first;
  v.u_rows = p->u_rows;
  v.pos = p->pos;
  v.marks = p->s_marks;
  v.base = p->base;
  v.rows = reinterpret_cast<uint32_t*>(p->rows);
  v.slice_rows = p->slice_rows;
  v.by_domain = p->by_domain ? 1u : 0u;
  // The drain instance stages no word table (two-level form), so its tensor-map parameter is free to carry the
  // view by value; place_ns_kernel static_asserts that the instance is two-level.
  CUtensorMap view;
  memset(&view, 0, sizeof(view));
  memcpy(&view, &v, sizeof(v));
  a.n_reqs = p->n_reqs;
  a.out = p->s_out;
  a.unpinned = p->s_unpinned;
  const size_t smem = ns_smem_bytes(l.word_rows, p->n_domains, false, false);
  static thread_local size_t attr_set = 0;
  if (smem > attr_set) {
    const cudaError_t e = cudaFuncSetAttribute(place_ns_kernel<false, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return -(int)e;
    attr_set = smem;
  }
  place_ns_kernel<false, true, true><<<p->grid, kNsThreads, smem, s>>>(a, view);
  return launch_result(3);
}

// The set-overlay solve of one drain placement waves step: the capacities and positions are those the drain
// placement's solve left (launch_place_ns_drain ran at setup); a persistent grid over the step's items.
int launch_place_ns_drain_set(const DrainPlaceWavesLaunch* d, int sm_count, cudaStream_t s) {
  const DrainPlaceLaunch* p = &d->p;
  const NsLayout l = ns_layout(p->n_nodes, p->n_domains, p->n_reqs, p->n_namespaces);
  if (p->round_bytes < l.total || p->n_reqs > 0xFFFFFFu) return -(int)cudaErrorInvalidValue;
  uint8_t* base = static_cast<uint8_t*>(p->round);
  PlaceNsArgs a{};
  a.nodes = p->nodes;
  a.reqs = p->reqs;
  a.occupancy = p->occupancy;
  a.dom_first = p->dom_first;
  a.node_order = p->node_order;
  a.g_words = reinterpret_cast<uint32_t*>(base + l.words);
  a.g_nodes2 = reinterpret_cast<uint32_t*>(base + l.nodes2);
  a.g_dom_free = reinterpret_cast<uint32_t*>(base + l.dom_free);
  a.ns_first = reinterpret_cast<uint32_t*>(base + l.ns_first);
  a.ns_rows = reinterpret_cast<uint32_t*>(base + l.ns_rows);
  a.ns_count = reinterpret_cast<uint32_t*>(base + l.ns_count);
  a.ns_cursor = reinterpret_cast<uint32_t*>(base + l.ns_cursor);
  a.counters = reinterpret_cast<uint32_t*>(base + l.counters) + 4u * 8u;
  a.n_nodes = p->n_nodes;
  a.n_domains = p->n_domains;
  a.n_namespaces = p->n_namespaces;
  a.n_parts = 1u;
  a.word_rows = l.word_rows;
  a.n_reqs = p->n_reqs;
  a.out = p->s_out;
  a.unpinned = p->s_unpinned;
  SetNsView v{};
  v.d.items = d->items;
  v.d.n_items = &d->st->n_items;
  v.d.item_capacity = d->item_capacity;
  v.d.u_first = p->u_first;
  v.d.u_rows = p->u_rows;
  v.d.pos = p->pos;
  v.d.marks = p->s_marks;
  v.d.base = p->base;
  v.d.rows = d->col_rows;
  v.d.slice_rows = p->slice_rows;
  v.d.by_domain = p->by_domain ? 1u : 0u;
  v.state = &d->st->key;
  v.u_wave = d->u_wave;
  v.key_wave = d->key_wave;
  v.drained = d->drained;
  CUtensorMap view;
  memset(&view, 0, sizeof(view));
  memcpy(&view, &v, sizeof(v));
  const size_t smem = ns_smem_bytes(l.word_rows, p->n_domains, false, false);
  static thread_local size_t attr_set = 0;
  if (smem > attr_set) {
    const cudaError_t e = cudaFuncSetAttribute(place_ns_kernel<false, true, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return -(int)e;
    attr_set = smem;
  }
  place_ns_kernel<false, true, true, true><<<p->grid, kNsThreads, smem, s>>>(a, view);
  return launch_result(1);
}

// The rollout instances' arguments over the round scratch, which holds the namespace index of every namespace.
static PlaceNsArgs rollout_ns_args(const RolloutPlaceLaunch* p, const NsLayout& l) {
  uint8_t* base = static_cast<uint8_t*>(p->round);
  PlaceNsArgs a{};
  a.nodes = p->nodes;
  a.reqs = p->reqs;
  a.occupancy = p->occupancy;
  a.dom_first = p->dom_first;
  a.node_order = p->node_order;
  a.g_words = reinterpret_cast<uint32_t*>(base + l.words);
  a.g_nodes2 = reinterpret_cast<uint32_t*>(base + l.nodes2);
  a.g_dom_free = reinterpret_cast<uint32_t*>(base + l.dom_free);
  a.ns_first = reinterpret_cast<uint32_t*>(base + l.ns_first);
  a.ns_rows = reinterpret_cast<uint32_t*>(base + l.ns_rows);
  a.ns_count = reinterpret_cast<uint32_t*>(base + l.ns_count);
  a.ns_cursor = reinterpret_cast<uint32_t*>(base + l.ns_cursor);
  a.counters = reinterpret_cast<uint32_t*>(base + l.counters) + 4u * 8u;  // a block no other call uses
  a.n_nodes = p->n_nodes;
  a.n_domains = p->n_domains;
  a.n_namespaces = p->n_namespaces;
  a.n_parts = 1u;
  a.word_rows = l.word_rows;
  return a;
}

static RollNsView rollout_ns_view(const RolloutPlaceLaunch* p) {
  RollNsView v{};
  v.d.items = p->items;
  v.d.n_items = p->counts;
  v.d.item_capacity = p->n;
  v.d.base = p->base;
  v.d.rows = p->rows_out;
  v.d.slice_rows = p->slice_rows;
  v.extra = p->extra;
  v.ent = p->ent;
  v.n_resident = p->n_reqs;
  return v;
}

// The rollout placement solve: the capacities of the node index (the condense kernel's part A alone), then the
// rollout instance over p->grid CTAs.  The round scratch holds the namespace index of every namespace.
int launch_place_ns_rollout(const RolloutPlaceLaunch* p, int sm_count, cudaStream_t s) {
  const NsLayout l = ns_layout(p->n_nodes, p->n_domains, p->n_reqs, p->n_namespaces);
  if (p->round_bytes < l.total || p->n_reqs > 0xFFFFFFu) return -(int)cudaErrorInvalidValue;
  PlaceNsArgs a = rollout_ns_args(p, l);
  {
    uint64_t grid = ((uint64_t)p->n_domains * 32u + 255) / 256;
    if (grid < 1) grid = 1;
    if (grid > (uint64_t)sm_count * 8u) grid = (uint64_t)sm_count * 8u;
    place_condense_kernel<<<(unsigned)grid, 256, 0, s>>>(a);  // (a.n_reqs = 0: capacities only)
    if (const int r = launch_result(0); r < 0) return r;
  }
  const RollNsView v = rollout_ns_view(p);
  CUtensorMap view;
  memset(&view, 0, sizeof(view));
  memcpy(&view, &v, sizeof(v));
  a.n_reqs = p->n_reqs;
  a.out = p->s_out;
  a.unpinned = p->s_unpinned;
  const size_t smem = ns_smem_bytes(l.word_rows, p->n_domains, false, false);
  static thread_local size_t attr_set = 0;
  if (smem > attr_set) {
    const cudaError_t e =
        cudaFuncSetAttribute(place_ns_kernel<false, true, true, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return -(int)e;
    attr_set = smem;
  }
  place_ns_kernel<false, true, true, false, true><<<p->grid, kNsThreads, smem, s>>>(a, view);
  return launch_result(2);
}

// One round's solve of the rollout waves: the wave instance over w->grid CTAs, on the capacities and the namespace
// index the setup's rollout solve left in the round scratch.
int launch_place_ns_rollout_wave(const RolloutPlaceWavesLaunch* w, cudaStream_t s) {
  const RolloutPlaceLaunch* p = &w->p;
  const NsLayout l = ns_layout(p->n_nodes, p->n_domains, p->n_reqs, p->n_namespaces);
  if (p->round_bytes < l.total || p->n_reqs > 0xFFFFFFu) return -(int)cudaErrorInvalidValue;
  PlaceNsArgs a = rollout_ns_args(p, l);
  RollWaveNsView v{};
  v.r = rollout_ns_view(p);
  v.r.d.items = w->items;
  v.r.d.n_items = w->st + 1;
  v.r.d.rows = w->res;
  v.r.d.slice_rows = w->slice_rows;
  v.desc = w->desc;
  v.col = w->col;
  CUtensorMap view;
  memset(&view, 0, sizeof(view));
  memcpy(&view, &v, sizeof(v));
  a.n_reqs = p->n_reqs;
  a.out = w->s_out;
  a.unpinned = w->s_unpinned;
  const size_t smem = ns_smem_bytes(l.word_rows, p->n_domains, false, false);
  static thread_local size_t attr_set = 0;
  if (smem > attr_set) {
    const cudaError_t e = cudaFuncSetAttribute(place_ns_kernel<false, true, true, false, true, true>,
                                               cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return -(int)e;
    attr_set = smem;
  }
  place_ns_kernel<false, true, true, false, true, true><<<w->grid, kNsThreads, smem, s>>>(a, view);
  return launch_result(1);
}

int launch_index_scan(uint32_t* d_count, uint32_t* d_first, uint32_t* d_cursor, uint32_t n, cudaStream_t s) {
  place_index_scan_kernel<<<1, kIndexScanThreads, 0, s>>>(IndexScanArgs{d_count, d_first, d_cursor, n});
  return launch_result(1);
}

// The what-if's diff against the baseline and its counts.  counts: [0] changed rows [1] lost [2] moved
// [3] gained (resident rows) [4] PLACED [5] UNSCHEDULABLE [6] CONFLICT (every row, extra rows included).
// Each warp reduces its counts before the one atomic per counter, and appends its changed rows with one
// atomic (rows at or beyond `capacity` are counted, not listed).
struct WhatIfDiffArgs {
  const lwse_place_out* before;  // n_resident
  const lwse_place_out* after;   // n_total
  uint32_t* rows;
  lwse_place_out* outs_before;
  lwse_place_out* outs_after;
  uint32_t* counts;
  uint32_t capacity, n_resident, n_total;
};

__global__ void __launch_bounds__(256) place_whatif_diff_kernel(const WhatIfDiffArgs a) {
  const uint32_t lane = threadIdx.x & 31u, stride = gridDim.x * blockDim.x;
  uint32_t c[6] = {0u, 0u, 0u, 0u, 0u, 0u};
  for (uint32_t base = (blockIdx.x * blockDim.x + threadIdx.x) & ~31u; base < a.n_total; base += stride) {
    const uint32_t r = base + lane;
    bool changed = false;
    uint4 v = make_uint4(0u, 0u, 0u, 0u), o = v;
    if (r < a.n_total) {
      v = __ldcg(reinterpret_cast<const uint4*>(a.after + r));
      c[3] += (v.z & LWSE_PLACE_PLACED) ? 1u : 0u;
      c[4] += (v.z & LWSE_PLACE_UNSCHEDULABLE) ? 1u : 0u;
      c[5] += (v.z & LWSE_PLACE_CONFLICT) ? 1u : 0u;
      if (r < a.n_resident) {
        o = __ldcg(reinterpret_cast<const uint4*>(a.before + r));
        changed = v.x != o.x || v.y != o.y || v.z != o.z || v.w != o.w;
        const bool was = (o.z & LWSE_PLACE_PLACED) != 0u, is = (v.z & LWSE_PLACE_PLACED) != 0u;
        c[0] += (was && !is) ? 1u : 0u;
        c[1] += (was && is && o.x != v.x) ? 1u : 0u;
        c[2] += (!was && is) ? 1u : 0u;
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
#pragma unroll
  for (int k = 0; k < 6; k++) {
    const uint32_t sum = __reduce_add_sync(0xFFFFFFFFu, c[k]);
    if (lane == 0 && sum) atomicAdd(a.counts + 1 + k, sum);
  }
}

int launch_place_whatif_diff(const lwse_place_out* d_before, const lwse_place_out* d_after, uint32_t n_resident, uint32_t n_total,
                             uint32_t* d_rows, lwse_place_out* d_outs_before, lwse_place_out* d_outs_after, uint32_t capacity,
                             uint32_t* d_counts, int sm_count, cudaStream_t s) {
  const WhatIfDiffArgs a{d_before, d_after, d_rows, d_outs_before, d_outs_after, d_counts, capacity, n_resident, n_total};
  uint64_t grid = ((uint64_t)n_total + 255) / 256;
  if (grid < 1) grid = 1;
  if (grid > (uint64_t)sm_count * 4u) grid = (uint64_t)sm_count * 4u;
  place_whatif_diff_kernel<<<(unsigned)grid, 256, 0, s>>>(a);
  return launch_result(1);
}

}  // namespace lwse
