// Placement round (sm_90a) — build-defined spec, see oracle/lwse_oracle_place.c
// and DESIGN.md "Placement (parity unpinned)".
//
// One kernel, one warp per request:
//   phase 0  the grid condenses the node table (16 B/node) and the occupancy vector into
//            one word per node (free slots | domain), stored in DOMAIN-SORTED position
//            (the static order is built when the node table is uploaded), accumulates the
//            per-domain free capacity, and pinned requests (leader already scheduled)
//            claim their domain with atomicMin on the 64-bit holder key; one barrier;
//   rounds   deferred acceptance: every request that does not hold a domain is taken by
//            one warp — level 1: its lanes stride over the domains (holder + capacity from
//            L2, all loads of a lane in flight together), redux to the winning domain;
//            level 2: the lanes score the nodes of that one domain (a contiguous run of
//            the sorted words); lane 0 claims with atomicMin — and one barrier per round.
//            Holder keys only ever decrease, so the fixed point is unique and equals the
//            sequential "ascending key takes its best free domain" statement of the
//            oracle.  A claim that found the domain empty is settled; any other outcome
//            leaves somebody without a domain and is counted, and the rounds end when a
//            round counted nothing.
// Small problems (the steady state: most leaders are scheduled, few groups are new) run
// as ONE thread-block cluster of 8 CTAs: the barriers are cluster barriers (hardware,
// cheap) instead of grid barriers through L2 (microseconds each), the launch is an
// ordinary one, and only 8 SMs are touched, so the sweep kernels of the same tick keep
// the rest of the GPU.  Bursts run the same code as a cooperative grid.
#include <cooperative_groups.h>

#include <cstdlib>

#include "lwse_device.cuh"
#include "lwse_launch.cuh"

namespace cg = cooperative_groups;


namespace lwse {

struct PlaceArgs {
  const lwse_node_rec* nodes;
  const lwse_place_req* reqs;
  const uint32_t* occupancy;  // nullable
  lwse_place_out* out;
  // static index of the node table (built by lwse_upload_nodes)
  const uint32_t* dom_first;   // n_domains + 1: run of domain d in the sorted order
  const uint32_t* node_order;  // sorted position -> node row (usable nodes only)
  const uint32_t* node_pos;    // node row -> sorted position, or LWSE_NONE
  unsigned long long* holder;  // n_namespaces x n_domains
  uint32_t* counters;          // [0..2] unsettled claims per round (rotating), [3] rounds, [4] unpinned requests
  uint32_t* g_sorted;          // condensed node words in sorted position
  uint32_t* g_dom_free;
  uint32_t* unpinned;          // indices of the unpinned requests (built in phase 0)
  unsigned long long* next_holder;  // the scratch half the NEXT call will use: reset here
  uint32_t* next_zero;         // its counters + domain capacities
  uint32_t next_zero_words;
  uint32_t n_nodes, n_domains, n_reqs, n_namespaces;
  uint32_t hold_stride;  // n_domains rounded up to even: holder rows are 16-byte aligned
  uint32_t* last_unpinned;  // scratch tail (never reset): the number of live unpinned requests of this call
  // gathered form (multi-GPU): `reqs` / `occupancy` point into part 0 of n_parts equally laid out
  // parts (one per rank, as all-gathered); request r lives in part r / reqs_per_part, and the
  // occupancy of a node is the sum over the parts
  uint32_t n_parts, reqs_per_part;
  uint64_t part_stride_bytes;
};

constexpr uint32_t kPlaceThreads = 512;
constexpr uint32_t kPlaceWarps = kPlaceThreads / 32;
constexpr uint32_t kClusterCtas = 8;
constexpr uint32_t kCacheQ = 4;  // requests per warp whose state lives in shared memory

__device__ __forceinline__ uint32_t mix32(uint32_t x) {
  x ^= x >> 16;
  x *= 0x85EBCA6Bu;
  x ^= x >> 13;
  x *= 0xC2B2AE35u;
  x ^= x >> 16;
  return x;
}

__device__ __forceinline__ unsigned long long place_key(const lwse_place_req& r, uint32_t index, bool pinned) {
  return ((unsigned long long)(pinned ? 0 : 1) << 63) | (((r.priority >> 25) & 0x7FFFFFFFFFull) << 24) |
         (unsigned long long)(index & 0xFFFFFFu);
}

__device__ __forceinline__ lwse_place_req load_req(const PlaceArgs& a, uint32_t r) {
  const lwse_place_req* p = a.reqs;
  if (a.n_parts > 1u) {
    const uint32_t part = r / a.reqs_per_part, j = r - part * a.reqs_per_part;
    p = reinterpret_cast<const lwse_place_req*>(reinterpret_cast<const uint8_t*>(a.reqs) +
                                                (uint64_t)part * a.part_stride_bytes) + j;
  } else {
    p += r;
  }
  const uint4 lo = ldg_keep(reinterpret_cast<const uint4*>(p)), hi = ldg_keep(reinterpret_cast<const uint4*>(p) + 1);
  lwse_place_req q;
  q.priority = u64_of(lo.x, lo.y);
  q.group_key = u64_of(lo.z, lo.w);
  q.group = hi.x;
  q.ns = hi.y;
  q.size = (int32_t)hi.z;
  q.leader_node = hi.w;
  return q;
}

__device__ __forceinline__ uint32_t load_occupancy(const PlaceArgs& a, uint32_t n) {
  if (!a.occupancy) return 0u;
  uint32_t occ = 0;
  for (uint32_t p = 0; p < a.n_parts; p++)
    occ += ldg_keep_u32(reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint8_t*>(a.occupancy) +
                                                           (uint64_t)p * a.part_stride_bytes) + n);
  return occ;
}

// phase timestamps (ns, %globaltimer) of CTA 0 for tuning: counters[16 + 2k, 16 + 2k + 1]
__device__ __forceinline__ void stamp(const PlaceArgs& a, uint32_t k) {
  if (blockIdx.x == 0 && threadIdx.x == 0 && k < 16u) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    a.counters[16 + 2 * k] = (uint32_t)t;
    a.counters[17 + 2 * k] = (uint32_t)(t >> 32);
  }
}

// A warp's view of one of its requests across the rounds.  Everything a later round needs that
// is not in here lives in the request's result row (domain, flags), which the warp rewrites at
// every proposal: at the fixed point the row is the result.
struct ReqCache {
  unsigned long long key;
  uint32_t r, ns, size, key_lo, key_hi, cur_dom, dead, pad;
};

// Split barrier: everything a CTA wrote (plain stores and atomics) before arrive is visible to
// every thread of the cluster / grid after wait.  The cluster barrier is a hardware barrier with
// release / acquire semantics at cluster scope; the grid form goes through L2.
template <bool kCluster>
__device__ __forceinline__ void barrier_arrive() {
  if constexpr (kCluster) asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
}
template <bool kCluster>
__device__ __forceinline__ void barrier_wait() {
  if constexpr (kCluster) {
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
  } else {
    __threadfence();
    cg::this_grid().sync();
  }
}

__device__ __forceinline__ void store_out(lwse_place_out* p, uint32_t d, uint32_t n, uint32_t flags, uint32_t score) {
  *reinterpret_cast<uint4*>(p) = make_uint4(d, n, flags, score);
}

// the domain a pinned request claims (its leader's node decides), or LWSE_NONE
__device__ __forceinline__ uint32_t pinned_domain(const PlaceArgs& a, const lwse_place_req& rq) {
  if (rq.ns >= a.n_namespaces || rq.leader_node >= a.n_nodes) return LWSE_NONE;
  const uint4 nr = ldg_keep(reinterpret_cast<const uint4*>(a.nodes + rq.leader_node));
  return (((nr.w >> 16) & LWSE_NODE_HAS_TOPOLOGY) && nr.z < a.n_domains) ? nr.z : LWSE_NONE;
}

// result of a pinned request; called once every pinned claim is in (pinned keys, bit 63 clear,
// are below every unpinned key: the holder of a pinned domain never changes afterwards)
__device__ __forceinline__ void write_pinned(const PlaceArgs& a, const lwse_place_req& rq, uint32_t r, uint32_t d) {
  uint32_t flags = LWSE_PLACE_PINNED;
  if (rq.ns >= a.n_namespaces) {
    flags |= LWSE_PLACE_UNSCHEDULABLE;
  } else if (d != LWSE_NONE) {
    const unsigned long long h = __ldcg(a.holder + (uint64_t)rq.ns * a.hold_stride + d);
    flags |= h == place_key(rq, r, true) ? LWSE_PLACE_PLACED : LWSE_PLACE_CONFLICT;
  }
  store_out(a.out + r, d, rq.leader_node, flags, 0u);
}

// 64 registers in either form: the round shares its SMs with the sweep kernels of the same tick,
// and a cluster is only scheduled once EVERY one of its CTAs has an SM with room — 16 K registers
// per 256-thread CTA fit next to three resident CTAs of the fused sweep kernel, 28 K did not
// (the tick then serialised).  (A 512 x 92 first version held three quarters of each register
// file and the sweep's group pass could not start next to it at all.)
template <bool kCluster>
__global__ void __launch_bounds__(kPlaceThreads, 2) place_kernel(const PlaceArgs a) {
  constexpr int kDomChunk = kCluster ? 4 : 3;  // level 1: domain pairs per lane whose loads are in flight together
  __shared__ ReqCache s_req[kPlaceWarps][kCacheQ];
  __shared__ uint32_t s_scan[32];
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  const uint32_t gtid = blockIdx.x * blockDim.x + tid, gsize = gridDim.x * blockDim.x;
  stamp(a, 0);
  // After a peer exchange the round is launched programmatically dependent on the push kernel: the
  // cluster is already resident when the parts arrive (no-op for an ordinary launch).
  pdl_wait_prior();

  // ---------------- phase 0: node words, domain capacities, pinned claims ----------------
  // (this scratch half was left clean — holders ~0, counters and capacities 0 — by the previous call)
  // Request gtid stays in registers until its result is written (the common case: no more
  // requests than threads); its loads are issued first, the node loads next, so that the two
  // dependent chains (request → leader's node row → claim, node row → capacity) overlap.
  lwse_place_req rq0{};
  const bool has0 = gtid < a.n_reqs;
  if (has0) rq0 = load_req(a, gtid);
  for (uint32_t base = gtid; base < a.n_nodes; base += 3u * gsize) {
    uint32_t pos[3], occ[3];
    uint4 nr[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
      const uint32_t n = base + (uint32_t)k * gsize;
      pos[k] = n < a.n_nodes ? ldg_keep_u32(a.node_pos + n) : LWSE_NONE;
      nr[k] = n < a.n_nodes ? ldg_keep(reinterpret_cast<const uint4*>(a.nodes + n)) : make_uint4(0, 0, 0, 0);
      occ[k] = n < a.n_nodes ? load_occupancy(a, n) : 0u;
    }
#pragma unroll
    for (int k = 0; k < 3; k++) {
      if (pos[k] == LWSE_NONE) continue;  // not schedulable / no topology label: no request can use it
      const uint32_t d = nr[k].z, cap = nr[k].w & 0xFFFFu;
      const uint32_t fr = cap > occ[k] ? cap - occ[k] : 0u;
      a.g_sorted[pos[k]] = (min(fr, 15u) << 28) | d;
      if (fr) atomicAdd(a.g_dom_free + d, fr);
    }
  }
  uint32_t d0 = LWSE_NONE;  // the domain request gtid claims, if it is pinned
  for (uint32_t base = 0; base < a.n_reqs; base += gsize) {  // uniform trip count: the CTA compacts together
    const uint32_t r = base + gtid;
    bool live_unpinned = false;
    if (r < a.n_reqs) {
      const lwse_place_req rq = r == gtid ? rq0 : load_req(a, r);
      if (rq.leader_node == LWSE_NONE) {
        const bool dead = rq.ns >= a.n_namespaces || rq.size < 1;
        store_out(a.out + r, LWSE_NONE, LWSE_NONE, dead ? LWSE_PLACE_UNSCHEDULABLE : 0u, 0u);
        live_unpinned = !dead;
      } else {
        const uint32_t d = pinned_domain(a, rq);
        if (r == gtid) d0 = d;
        if (d != LWSE_NONE) atomicMin(a.holder + (uint64_t)rq.ns * a.hold_stride + d, place_key(rq, r, true));
      }
    }
    // the list of live unpinned requests: one atomic per CTA (a hundred same-address atomics
    // with a result serialise in L2); the order is irrelevant, the fixed point is unique
    const uint32_t ballot = __ballot_sync(0xFFFFFFFFu, live_unpinned);
    if (lane == 0) s_scan[warp] = __popc(ballot);
    __syncthreads();
    if (warp == 0) {
      const uint32_t mine = lane < (blockDim.x >> 5) ? s_scan[lane] : 0u;
      uint32_t incl = mine;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const uint32_t v = __shfl_up_sync(0xFFFFFFFFu, incl, off);
        if ((int)lane >= off) incl += v;
      }
      const uint32_t total = __shfl_sync(0xFFFFFFFFu, incl, 31);
      uint32_t cta_base = 0;
      if (lane == 0 && total) cta_base = atomicAdd(a.counters + 4, total);
      cta_base = __shfl_sync(0xFFFFFFFFu, cta_base, 0);
      if (lane < (blockDim.x >> 5)) s_scan[lane] = cta_base + incl - mine;
    }
    __syncthreads();
    if (live_unpinned) a.unpinned[s_scan[warp] + __popc(ballot & ((1u << lane) - 1u))] = r;
    __syncthreads();  // s_scan is reused by the next pass
  }
  // leave the other scratch half clean for the next call (it is idle: calls are stream-ordered)
  {
    const uint64_t n_hold = (uint64_t)a.n_namespaces * a.hold_stride;
    for (uint64_t i = gtid; i < n_hold; i += gsize) a.next_holder[i] = ~0ull;
    for (uint32_t i = gtid; i < a.next_zero_words; i += gsize) a.next_zero[i] = 0u;
  }
  stamp(a, 1);
  barrier_arrive<kCluster>();
  barrier_wait<kCluster>();
  stamp(a, 2);

  // results of the pinned requests (final as of now); the cluster form writes them while it
  // waits at the first round barrier instead
  auto pinned_results = [&]() {
    for (uint32_t r = gtid; r < a.n_reqs; r += gsize) {
      if (r == gtid) {
        if (rq0.leader_node != LWSE_NONE) write_pinned(a, rq0, r, d0);
      } else {
        const lwse_place_req rq = load_req(a, r);
        if (rq.leader_node != LWSE_NONE) write_pinned(a, rq, r, pinned_domain(a, rq));
      }
    }
  };
  const uint32_t n_unpinned = __ldcg(a.counters + 4);
  if (gtid == 0) *a.last_unpinned = n_unpinned;
  if (!kCluster || n_unpinned == 0u) pinned_results();

  uint32_t round = 0;
  if (n_unpinned) {
    // this warp's requests: k = gw, gw + GW, …  (warp-major across the CTAs, so that few requests
    // spread over all the CTAs); the first kCacheQ live in shared memory
    const uint32_t GW = gridDim.x * (blockDim.x >> 5), gw = warp * gridDim.x + blockIdx.x;
    const uint32_t my_count = gw < n_unpinned ? (n_unpinned - gw + GW - 1u) / GW : 0u;
    auto load_cache = [&](uint32_t j) {
      const uint32_t r = __ldcg(a.unpinned + gw + j * GW);
      const lwse_place_req rq = load_req(a, r);
      ReqCache q;
      q.key = place_key(rq, r, false);
      q.r = r;
      q.ns = rq.ns;
      q.size = (uint32_t)rq.size;
      q.key_lo = (uint32_t)rq.group_key;
      q.key_hi = (uint32_t)(rq.group_key >> 32);
      q.cur_dom = LWSE_NONE;
      q.dead = 0;
      q.pad = 0;
      return q;
    };
    if (lane < min(my_count, kCacheQ)) s_req[warp][lane] = load_cache(lane);
    __syncwarp();
    stamp(a, 3);

    // ---------------- deferred-acceptance rounds, one warp per request ----------------
    for (;; round++) {
      // three rotating counters: the one for round k+1 is cleared during round k,
      // when nobody can still be reading it (it was last read after round k-2)
      uint32_t* counter = a.counters + (round % 3u);
      if (gtid == 0) a.counters[(round + 1u) % 3u] = 0;
      for (uint32_t j = 0; j < my_count; j++) {
        ReqCache q;
        if (j < kCacheQ) {
          q = s_req[warp][j];
        } else {  // overflow: the state lives in the result row (written by this warp only)
          q = load_cache(j);
          const uint4 o = __ldcg(reinterpret_cast<const uint4*>(a.out + q.r));
          q.cur_dom = o.x;
          q.dead = (o.z & LWSE_PLACE_UNSCHEDULABLE) ? 1u : 0u;
        }
        __syncwarp();  // every lane has its copy before lane 0 updates the cache entry below
        if (q.dead) continue;  // warp-uniform
        const unsigned long long key = q.key;
        unsigned long long* hold = a.holder + (uint64_t)q.ns * a.hold_stride;
        // Level 1 — the domain.  A lane takes domain pairs (2 lane, 2 lane + 1), (+64, …): one
        // 16-byte load of two holders and one 8-byte load of two capacities per pair, kDomChunk
        // pairs in flight together.  Holders change under our feet during a round (other warps'
        // atomicMin); a stale reading can only make a proposal fail, never skip a domain that is
        // free (holder keys only decrease), and a failed proposal is counted and repeated.
        // (Out-of-range slots need no test: their capacity reads as 0 — a skipped pair, or the
        // zero word after the last domain — so their score is 0.)
        if (q.cur_dom != LWSE_NONE && __ldcg(hold + q.cur_dom) == key) continue;  // still holds what it proposed to
        uint32_t my_hi = 0, my_d = LWSE_NONE;
        for (uint32_t c0 = 2u * lane; c0 < a.n_domains; c0 += 64u * kDomChunk) {
          ulonglong2 h[kDomChunk];
          uint2 cap[kDomChunk];
#pragma unroll
          for (int k = 0; k < kDomChunk; k++) {
            const uint32_t d = c0 + 64u * (uint32_t)k;
            if (d < a.n_domains) {
              h[k] = __ldcg(reinterpret_cast<const ulonglong2*>(hold + d));
              cap[k] = __ldcg(reinterpret_cast<const uint2*>(a.g_dom_free + d));
            } else {
              h[k] = make_ulonglong2(0ull, 0ull);
              cap[k] = make_uint2(0u, 0u);
            }
          }
          uint32_t hi[2 * kDomChunk];  // independent chains first, one max-reduction after
#pragma unroll
          for (int k = 0; k < kDomChunk; k++) {
            const uint32_t d = c0 + 64u * (uint32_t)k;
            const uint32_t m0 = mix32(q.key_lo ^ (d * 0x9E3779B1u)) | 1u;
            const uint32_t m1 = mix32(q.key_lo ^ ((d + 1u) * 0x9E3779B1u)) | 1u;
            hi[2 * k] = (cap[k].x >= q.size && h[k].x >= key) ? m0 : 0u;
            hi[2 * k + 1] = (cap[k].y >= q.size && h[k].y >= key) ? m1 : 0u;
          }
#pragma unroll
          for (int k = 0; k < 2 * kDomChunk; k++) {  // slot order = ascending domain: ties keep the lower one
            const uint32_t d = c0 + 64u * (uint32_t)(k >> 1) + (uint32_t)(k & 1);
            const bool better = hi[k] > my_hi;
            my_hi = better ? hi[k] : my_hi;
            my_d = better ? d : my_d;
          }
        }
        const uint32_t H = __reduce_max_sync(0xFFFFFFFFu, my_hi);
        if (H == 0u) {  // nothing feasible now, and the feasible set only shrinks
          if (lane == 0) {
            store_out(a.out + q.r, LWSE_NONE, LWSE_NONE, LWSE_PLACE_UNSCHEDULABLE, 0u);
            if (j < kCacheQ) s_req[warp][j].dead = 1u;
          }
          __syncwarp();
          continue;
        }
        const uint32_t best_d = __reduce_min_sync(0xFFFFFFFFu, my_hi == H ? my_d : LWSE_NONE);
        // Level 2 — the node: the domain's run of the sorted node words.
        const uint32_t first = ldg_keep_u32(a.dom_first + best_d), last = ldg_keep_u32(a.dom_first + best_d + 1u);
        uint32_t my_lo = 0, my_n = LWSE_NONE;
        for (uint32_t i = first + lane; i < last; i += 32u) {
          const uint32_t w = __ldcg(a.g_sorted + i);
          const uint32_t n = ldg_keep_u32(a.node_order + i);
          if ((w >> 28) == 0u) continue;
          const uint32_t lo = ((w >> 28) << 28) | (mix32(q.key_hi ^ (n * 0x85EBCA77u)) >> 4);
          if (lo > my_lo || (lo == my_lo && n < my_n)) {
            my_lo = lo;
            my_n = n;
          }
        }
        const uint32_t L = __reduce_max_sync(0xFFFFFFFFu, my_lo);
        const uint32_t best_n = __reduce_min_sync(0xFFFFFFFFu, (my_lo == L && L != 0u) ? my_n : LWSE_NONE);
        if (lane == 0) {
          if (best_n == LWSE_NONE) {  // cannot happen (capacity >= size >= 1 means a node with a free slot)
            store_out(a.out + q.r, LWSE_NONE, LWSE_NONE, LWSE_PLACE_UNSCHEDULABLE, 0u);
            if (j < kCacheQ) s_req[warp][j].dead = 1u;
          } else {
            store_out(a.out + q.r, best_d, best_n, LWSE_PLACE_PLACED, H);
            if (j < kCacheQ) s_req[warp][j].cur_dom = best_d;
            // A claim on an empty domain settles at once.  Any other outcome leaves somebody
            // without a domain — the previous holder (old > key) or this request (old < key) —
            // who proposes again next round: count it.
            const unsigned long long old = atomicMin(hold + best_d, key);
            if (old != ~0ull) atomicAdd(counter, 1u);
          }
        }
        __syncwarp();
      }
      stamp(a, 4 + 2 * round);
      barrier_arrive<kCluster>();
      if (kCluster && round == 0u) pinned_results();  // off the critical path: the slowest warp is still proposing
      barrier_wait<kCluster>();
      stamp(a, 5 + 2 * round);
      const uint32_t unsettled = __ldcg(counter);
      if (unsettled == 0u || round > a.n_reqs + 2u) break;
    }
  }
  if (gtid == 0) a.counters[3] = n_unpinned ? round + 1u : 0u;
  stamp(a, 15);
}

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// scratch: two identical halves used alternately by successive calls; each half is
// [holder | counters(256 B) | g_dom_free | unpinned | g_sorted].  A call resets the
// holders / counters / capacities of the *other* half, so no memset sits on the critical path
// (the engine zero-fills the whole scratch once, when it allocates it).
static uint32_t hold_stride_of(uint32_t n_domains) { return (n_domains + 1u) & ~1u; }
static size_t place_half_bytes(uint32_t n_nodes, uint32_t n_domains, uint32_t n_reqs, uint32_t n_namespaces) {
  return align_up((size_t)n_namespaces * hold_stride_of(n_domains) * 8, 256) + 256 + align_up((size_t)n_domains * 4 + 16, 256) +
         align_up((size_t)n_reqs * 4, 256) + align_up((size_t)n_nodes * 4 + 128, 256);
}
size_t place_scratch_bytes(uint32_t n_nodes, uint32_t n_domains, uint32_t n_reqs, uint32_t n_namespaces) {
  return 2 * place_half_bytes(n_nodes, n_domains, n_reqs, n_namespaces) + 1024;
}

// `fresh`: the scratch was (re)allocated or its geometry changed → initialise both halves first.
int launch_place(const lwse_node_rec* d_nodes, const uint32_t* d_dom_first, const uint32_t* d_node_order,
                 const uint32_t* d_node_pos, uint32_t n_nodes, uint32_t n_domains, const lwse_place_req* d_reqs,
                 uint32_t n_reqs, const uint32_t* d_occupancy, uint32_t n_namespaces, lwse_place_out* d_out,
                 void* d_scratch, size_t scratch_bytes, uint32_t* h_rounds, int sm_count, cudaStream_t s,
                 uint32_t call_index, bool fresh, uint32_t n_parts, uint32_t reqs_per_part, uint64_t part_stride_bytes,
                 uint32_t* h_unpinned, const uint32_t** d_counters_out, const uint32_t** d_unpinned_out, bool after_push) {
  if (n_reqs > 0xFFFFFFu || n_domains >= (1u << 28) ||
      scratch_bytes < place_scratch_bytes(n_nodes, n_domains, n_reqs, n_namespaces))
    return -(int)cudaErrorInvalidValue;
  const size_t half = place_half_bytes(n_nodes, n_domains, n_reqs, n_namespaces);
  const size_t holder_bytes = align_up((size_t)n_namespaces * hold_stride_of(n_domains) * 8, 256);
  const size_t zero_bytes = 256 + align_up((size_t)n_domains * 4 + 16, 256);
  uint8_t* base = static_cast<uint8_t*>(d_scratch);
  uint8_t* p = base + (call_index & 1u) * half;
  uint8_t* q = base + ((call_index + 1u) & 1u) * half;
  cudaError_t e = cudaSuccess;
  if (fresh) {
    for (int h = 0; h < 2 && e == cudaSuccess; h++) {
      e = cudaMemsetAsync(base + h * half, 0xFF, holder_bytes, s);
      if (e == cudaSuccess) e = cudaMemsetAsync(base + h * half + holder_bytes, 0, zero_bytes, s);
    }
    if (e != cudaSuccess) return -(int)e;
  }
  PlaceArgs a{};
  a.nodes = d_nodes;
  a.reqs = d_reqs;
  a.occupancy = d_occupancy;
  a.out = d_out;
  a.dom_first = d_dom_first;
  a.node_order = d_node_order;
  a.node_pos = d_node_pos;
  a.holder = reinterpret_cast<unsigned long long*>(p);
  a.next_holder = reinterpret_cast<unsigned long long*>(q);
  p += holder_bytes;
  q += holder_bytes;
  a.counters = reinterpret_cast<uint32_t*>(p);
  a.g_dom_free = reinterpret_cast<uint32_t*>(p + 256);
  a.next_zero = reinterpret_cast<uint32_t*>(q);
  a.next_zero_words = (uint32_t)(zero_bytes / 4);
  p += zero_bytes;
  a.unpinned = reinterpret_cast<uint32_t*>(p);
  p += align_up((size_t)n_reqs * 4, 256);
  a.g_sorted = reinterpret_cast<uint32_t*>(p);
  a.n_nodes = n_nodes;
  a.n_domains = n_domains;
  a.n_reqs = n_reqs;
  a.n_namespaces = n_namespaces;
  a.hold_stride = hold_stride_of(n_domains);
  a.n_parts = n_parts ? n_parts : 1u;
  a.reqs_per_part = reqs_per_part ? reqs_per_part : n_reqs;
  a.part_stride_bytes = part_stride_bytes;
  a.last_unpinned = reinterpret_cast<uint32_t*>(base + 2 * half);
  if (d_counters_out) *d_counters_out = a.counters;       // phase stamps of this call (tuning aid)
  if (d_unpinned_out) *d_unpinned_out = a.last_unpinned;  // where this call leaves its unpinned-request count

  // One cluster while every request can have its own warp within a few passes; beyond that a
  // cooperative grid with one warp per request, at most one CTA per SM.
  // (phase 0 and the scratch reset are grid-stride loops: tables that 4096 threads cannot sweep in
  // a few passes go to the grid as well.)  What decides is the number of UNPINNED requests — pinned
  // ones cost one claim in phase 0 — and the host does not know it: the previous call's count,
  // copied to pinned host memory off the critical path by the engine, predicts this call's (no
  // history: all requests).  (The kernel does not post the count to mapped host memory itself:
  // the grid would not retire before the PCIe write is flushed.)
  const bool few_reqs = n_reqs <= kClusterCtas * kPlaceWarps * 8u;  // ≤ 8 per warp even if all are unpinned
  const uint32_t expect_unpinned = (!fresh && h_unpinned && *(volatile uint32_t*)h_unpinned != 0xFFFFFFFFu)
                                       ? *(volatile uint32_t*)h_unpinned
                                       : n_reqs;
  const bool small = (few_reqs || (expect_unpinned <= kClusterCtas * kPlaceWarps * 2u && n_reqs <= (1u << 14))) &&
                     n_nodes <= (1u << 16) && (uint64_t)n_namespaces * hold_stride_of(n_domains) <= (1u << 16);
  if (small) {
    // 16 CTAs x 256 threads where the device can co-schedule a 16-CTA cluster (non-portable size:
    // probed once per device), else 8 x 512: the same 128 warps on twice the SMs — the rounds are
    // bound by the instruction issue of the warps sharing a scheduler.
    // (function attributes are per device: probe once per device this process launches on)
    static int wide_by_device[64];  // 0 = not probed, 1 = 8 x 512, 2 = 16 x 256
    int dev = 0;
    cudaGetDevice(&dev);
    int& probed = wide_by_device[dev & 63];
    if (probed == 0) {
      probed = 1;
      if (cudaFuncSetAttribute(place_kernel<true>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) == cudaSuccess) {
        cudaLaunchConfig_t probe{};
        probe.gridDim = dim3(16);
        probe.blockDim = dim3(256);
        cudaLaunchAttribute pa[1];
        pa[0].id = cudaLaunchAttributeClusterDimension;
        pa[0].val.clusterDim.x = 16;
        pa[0].val.clusterDim.y = 1;
        pa[0].val.clusterDim.z = 1;
        probe.attrs = pa;
        probe.numAttrs = 1;
        int n = 0;
        if (cudaOccupancyMaxActiveClusters(&n, place_kernel<true>, &probe) == cudaSuccess && n >= 1) probed = 2;
      }
      (void)cudaGetLastError();
    }
    const int wide = probed == 2;
    const unsigned cl = wide ? 16u : kClusterCtas;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(cl);
    cfg.blockDim = dim3(wide ? 256u : kPlaceThreads);
    cfg.stream = s;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = cl;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = after_push ? 2 : 1;
    e = cudaLaunchKernelEx(&cfg, place_kernel<true>, a);
  } else {
    unsigned ctas = (n_reqs + kPlaceWarps - 1u) / kPlaceWarps;
    if (ctas > (unsigned)sm_count) ctas = (unsigned)sm_count;
    if (ctas < 16u) ctas = 16u;
    void* params[] = {&a};
    e = cudaLaunchCooperativeKernel((const void*)place_kernel<false>, dim3(ctas), dim3(kPlaceThreads), params, 0, s);
  }
  if (e != cudaSuccess) return -(int)e;
  if (h_rounds) {
    e = cudaMemcpyAsync(h_rounds, a.counters + 3, sizeof(uint32_t), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) return -(int)e;
  }
  return 1;
}

// --------------------------------------------------------------------------
// tick: which placement rows changed
// --------------------------------------------------------------------------
// Runs right after the placement kernel of a resident tick (programmatically dependent on it):
// result rows that differ from the previous tick's are appended to a device-memory change list
// and the previous-result table is brought up to date.  The tick's publish kernel
// (lwse_lws_kernels.cu) then moves the list to the host.
struct PlaceDiffArgs {
  const lwse_place_out* cur;
  lwse_place_out* prev;
  uint32_t n;
  uint32_t* rows;        // device list
  lwse_place_out* outs;
  uint32_t capacity;
  uint32_t* d_count;
};

__global__ void __launch_bounds__(256) place_diff_kernel(const PlaceDiffArgs a) {
  pdl_launch_dependents();
  pdl_wait_prior();
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < a.n; r += gridDim.x * blockDim.x) {
    const uint4 v = __ldcg(reinterpret_cast<const uint4*>(a.cur + r));
    const uint4 o = __ldcg(reinterpret_cast<const uint4*>(a.prev + r));
    if (v.x != o.x || v.y != o.y || v.z != o.z || v.w != o.w) {
      const uint32_t i = atomicAdd(a.d_count, 1u);
      if (i < a.capacity) {
        a.rows[i] = r;
        *reinterpret_cast<uint4*>(a.outs + i) = v;
      }
      *reinterpret_cast<uint4*>(a.prev + r) = v;
    }
  }
}

int launch_place_diff(const lwse_place_out* d_cur, lwse_place_out* d_prev, uint32_t n, uint32_t* d_rows,
                      lwse_place_out* d_outs, uint32_t capacity, uint32_t* d_count, cudaStream_t s) {
  PlaceDiffArgs a{d_cur, d_prev, n, d_rows, d_outs, capacity, d_count};
  unsigned grid = (n + 255u) / 256u;
  if (grid < 1u) grid = 1u;
  if (grid > (unsigned)kSmCount * 4u) grid = (unsigned)kSmCount * 4u;
  const cudaError_t e = launch_pdl(place_diff_kernel, dim3(grid), dim3(256), 0, s, true, a);
  if (e != cudaSuccess) return -(int)e;
  return 1;
}

}  // namespace lwse
