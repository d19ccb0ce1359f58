// Placement explanation (lwse_resident_place_explain, sm_90a); the definition is in lwse.h, the argument in DESIGN.md
// §3.5 ("The placement explanation").  Over one round — the baseline's node, request and result rows read in place,
// or a what-if round's scratch:
//
//   place_explain_stats_kernel   a thread per node row: dom_free, usable and free_all per domain, one atomic per
//                                counter per domain run of a warp (__match_any_sync).
//   by mask: place_explain_count_kernel (the selected rows of each 256-row chunk), place_index_scan_kernel (chunk
//            offsets), place_explain_fill_kernel (the rows in ascending order, their namespaces marked);
//   by list: place_explain_mark_kernel (the listed rows' namespaces marked).
//   place_explain_hold_kernel    a thread per result row: every PLACED row of a marked namespace atomicMin's its
//                                spec key into a linear-probing (namespace, domain) table.
//   place_explain_kernel         a warp per listed row: lanes stride the domains, classify them (the table is probed
//                                only for fitting domains), reduce the counts and the (hi, lower d) argmaxes; one
//                                atomic per warp per total.
#include "lwse_device.cuh"
#include "lwse_launch.cuh"

namespace lwse {

constexpr uint32_t kExplainChunk = 256;  // rows per count / fill block
constexpr unsigned long long kExplainEmpty = ~0ull;

__device__ __forceinline__ uint32_t explain_mix(uint32_t x) {  // the spec's mixer (murmur3 finalizer)
  x ^= x >> 16;
  x *= 0x85EBCA6Bu;
  x ^= x >> 13;
  x *= 0xC2B2AE35u;
  x ^= x >> 16;
  return x;
}

__device__ __forceinline__ unsigned long long explain_key(const lwse_place_req& r, uint32_t row) {
  const bool pinned = r.leader_node != LWSE_NONE;
  return ((unsigned long long)(pinned ? 0 : 1) << 63) | (((r.priority >> 25) & 0x7FFFFFFFFFull) << 24) |
         (unsigned long long)(row & 0xFFFFFFu);
}

__device__ __forceinline__ uint32_t explain_slot(unsigned long long k, uint32_t mask) {
  k ^= k >> 33;
  k *= 0xFF51AFD7ED558CCDull;
  k ^= k >> 33;
  return (uint32_t)k & mask;
}

// The holder's key of (ns, d), kExplainEmpty when nobody holds it.
__device__ __forceinline__ unsigned long long explain_holder(const PlaceExplainLaunch& p, uint32_t ns, uint32_t d) {
  const unsigned long long k = (unsigned long long)ns << 32 | d;
  uint32_t h = explain_slot(k, p.table_mask);
  for (uint32_t probe = 0; probe <= p.table_mask; probe++, h = (h + 1u) & p.table_mask) {
    const unsigned long long t = p.tkeys[h];
    if (t == k) return p.tvals[h];
    if (t == kExplainEmpty) break;
  }
  return kExplainEmpty;
}

__global__ void __launch_bounds__(256) place_explain_stats_kernel(const PlaceExplainLaunch p) {
  const uint32_t lane = threadIdx.x & 31u, stride = gridDim.x * blockDim.x;
  uint32_t* dom_free = p.dom;
  uint32_t* usable = p.dom + p.n_domains;
  uint32_t* free_all = p.dom + 2u * p.n_domains;
  for (uint32_t base = (blockIdx.x * blockDim.x + threadIdx.x) & ~31u; base < p.n_nodes; base += stride) {
    const uint32_t n = base + lane;
    uint32_t d = LWSE_NONE, fr = 0, us = 0;
    if (n < p.n_nodes) {
      const uint4 nr = __ldg(reinterpret_cast<const uint4*>(p.nodes + n));
      const uint32_t flags = nr.w >> 16, cap = nr.w & 0xFFFFu;
      if ((flags & LWSE_NODE_HAS_TOPOLOGY) && nr.z < p.n_domains) {
        const uint32_t occ = p.occupancy ? __ldg(p.occupancy + n) : 0u;
        d = nr.z;
        fr = cap > occ ? cap - occ : 0u;
        us = (flags & LWSE_NODE_SCHEDULABLE) ? 1u : 0u;
      }
    }
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, d);
    if (d != LWSE_NONE) {
      const uint32_t all = __reduce_add_sync(peers, fr), use = __reduce_add_sync(peers, us ? fr : 0u);
      const uint32_t cnt = __reduce_add_sync(peers, us);
      if (lane == (uint32_t)__ffs(peers) - 1u) {
        if (use) atomicAdd(dom_free + d, use);
        if (cnt) atomicAdd(usable + d, cnt);
        if (all) atomicAdd(free_all + d, all);
      }
    }
  }
}

__device__ __forceinline__ bool explain_selected(const PlaceExplainLaunch& p, uint32_t i) {
  return i < p.n_rows && (__ldg(&p.res[i].flags) & p.mask) != 0u;
}

__device__ __forceinline__ void explain_mark(const PlaceExplainLaunch& p, uint32_t i) {
  const uint32_t v = __ldg(&p.reqs[i].ns);
  if (v < p.n_namespaces) p.ns_mark[v] = 1u;
}

__global__ void __launch_bounds__(kExplainChunk) place_explain_count_kernel(const PlaceExplainLaunch p) {
  const uint32_t n_chunks = (p.n_rows + kExplainChunk - 1u) / kExplainChunk;
  for (uint32_t b = blockIdx.x; b < n_chunks; b += gridDim.x) {
    const uint32_t c = (uint32_t)__syncthreads_count(explain_selected(p, b * kExplainChunk + threadIdx.x));
    if (threadIdx.x == 0) p.chunk_count[b] = c;
  }
}

__global__ void __launch_bounds__(kExplainChunk) place_explain_fill_kernel(const PlaceExplainLaunch p) {
  __shared__ uint32_t s_warp[kExplainChunk / 32];
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint32_t n_chunks = (p.n_rows + kExplainChunk - 1u) / kExplainChunk;
  for (uint32_t b = blockIdx.x; b < n_chunks; b += gridDim.x) {
    const uint32_t i = b * kExplainChunk + threadIdx.x;
    const bool sel = explain_selected(p, i);
    const uint32_t bal = __ballot_sync(0xFFFFFFFFu, sel);
    if (lane == 0) s_warp[warp] = (uint32_t)__popc(bal);
    __syncthreads();
    uint32_t at = __ldcg(p.chunk_first + b);
    for (uint32_t w = 0; w < warp; w++) at += s_warp[w];
    if (sel) {
      p.list[at + (uint32_t)__popc(bal & ((1u << lane) - 1u))] = i;
      explain_mark(p, i);
    }
    __syncthreads();  // s_warp is read before the next chunk writes it
  }
}

__global__ void __launch_bounds__(256) place_explain_mark_kernel(const PlaceExplainLaunch p) {
  const uint32_t n = __ldcg(p.n_list);
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) explain_mark(p, __ldcg(p.list + k));
}

__global__ void __launch_bounds__(256) place_explain_hold_kernel(const PlaceExplainLaunch p) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < p.n_rows; i += gridDim.x * blockDim.x) {
    const uint4 o = __ldg(reinterpret_cast<const uint4*>(p.res + i));
    if (!(o.z & LWSE_PLACE_PLACED) || o.x >= p.n_domains) continue;
    const lwse_place_req r = p.reqs[i];
    if (r.ns >= p.n_namespaces || !__ldcg(p.ns_mark + r.ns)) continue;
    const unsigned long long k = (unsigned long long)r.ns << 32 | o.x;
    uint32_t h = explain_slot(k, p.table_mask);
    for (uint32_t probe = 0; probe <= p.table_mask; probe++, h = (h + 1u) & p.table_mask) {
      const unsigned long long prev = atomicCAS(p.tkeys + h, kExplainEmpty, k);
      if (prev == kExplainEmpty || prev == k) {
        atomicMin(p.tvals + h, explain_key(r, i));
        break;
      }
    }
  }
}

// (hi, lower d) as one word: the larger word has the larger hash, then the lower domain; 0 = none.
__device__ __forceinline__ unsigned long long explain_pack(uint32_t hi, uint32_t d) {
  return (unsigned long long)hi << 32 | (0xFFFFFFFFu - d);
}

__device__ __forceinline__ unsigned long long warp_max_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long y = __shfl_xor_sync(0xFFFFFFFFu, v, o);
    v = y > v ? y : v;
  }
  return v;
}

__device__ __forceinline__ unsigned long long warp_min_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long y = __shfl_xor_sync(0xFFFFFFFFu, v, o);
    v = y < v ? y : v;
  }
  return v;
}

// Counts in c[]: the seven classes, fit_uncordoned, then the fitting domains.
enum : uint32_t { kOwn, kNoUsable, kTooSmall, kHeldPinned, kHeldEarlier, kHeldLater, kOpen, kFitUncordoned, kFit, kCounts };

__global__ void __launch_bounds__(256) place_explain_kernel(const PlaceExplainLaunch p) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t gwarp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t n = __ldcg(p.n_list);
  const uint32_t* dom_free = p.dom;
  const uint32_t* usable = p.dom + p.n_domains;
  const uint32_t* free_all = p.dom + 2u * p.n_domains;
  for (uint32_t k = gwarp; k < n; k += n_warps) {
    const uint32_t r = __ldcg(p.list + k);
    const lwse_place_req q = p.reqs[r];
    const uint32_t place_flags = __ldg(&p.res[r].flags), own = (place_flags & LWSE_PLACE_PLACED) ? __ldg(&p.res[r].domain_id) : LWSE_NONE;
    const bool pinned = q.leader_node != LWSE_NONE;
    const unsigned long long key = explain_key(q, r);
    const long long s = q.size;
    uint32_t c[kCounts] = {};
    uint32_t flags = 0, best_d = LWSE_NONE, blk_d = LWSE_NONE, blk_row = LWSE_NONE, short_d = LWSE_NONE, short_v = 0;
    if (q.ns >= p.n_namespaces) {
      flags = LWSE_PEX_NO_NAMESPACE;
    } else {
      const uint32_t key_lo = (uint32_t)q.group_key;
      unsigned long long best = 0, blk = 0, shortest = ~0ull;
      uint32_t my_blk_row = LWSE_NONE;
      for (uint32_t d = lane; d < p.n_domains; d += 32u) {
        const uint32_t df = __ldg(dom_free + d), us = __ldg(usable + d), fa = __ldg(free_all + d);
        const bool fits = us > 0u && (long long)df >= s;
        c[kFit] += fits ? 1u : 0u;
        if (d == own) {
          c[kOwn]++;
          best = max(best, explain_pack(explain_mix(key_lo ^ (d * 0x9E3779B1u)) | 1u, d));
        } else if (!fits) {
          if (us == 0u) {
            c[kNoUsable]++;
          } else {
            c[kTooSmall]++;
            shortest = min(shortest, (unsigned long long)(uint32_t)(s - (long long)df) << 32 | d);
          }
          if ((long long)fa >= s) c[kFitUncordoned]++;
        } else {
          const unsigned long long hk = explain_holder(p, q.ns, d);
          const unsigned long long w = explain_pack(explain_mix(key_lo ^ (d * 0x9E3779B1u)) | 1u, d);
          if (hk == kExplainEmpty) {
            c[kOpen]++;
            best = max(best, w);
          } else if (hk < key) {
            c[(hk >> 63) ? kHeldEarlier : kHeldPinned]++;
            if (w > blk) {
              blk = w;
              my_blk_row = (uint32_t)(hk & 0xFFFFFFu);
            }
          } else {
            c[kHeldLater]++;
            best = max(best, w);
          }
        }
      }
#pragma unroll
      for (uint32_t j = 0; j < kCounts; j++) c[j] = __reduce_add_sync(0xFFFFFFFFu, c[j]);
      best = warp_max_u64(best);
      const unsigned long long blk_all = warp_max_u64(blk);
      shortest = warp_min_u64(shortest);
      if (best) best_d = 0xFFFFFFFFu - (uint32_t)best;
      if (blk_all) {
        blk_d = 0xFFFFFFFFu - (uint32_t)blk_all;
        const uint32_t owner = (uint32_t)__ffs(__ballot_sync(0xFFFFFFFFu, blk == blk_all)) - 1u;
        blk_row = __shfl_sync(0xFFFFFFFFu, my_blk_row, (int)owner);
      }
      if (shortest != ~0ull) {
        short_d = (uint32_t)shortest;
        short_v = (uint32_t)(shortest >> 32);
      }
      if (c[kFit] == 0u) flags |= LWSE_PEX_CAPACITY;
      if (c[kFit] > 0u && c[kHeldPinned] + c[kHeldEarlier] == c[kFit]) flags |= LWSE_PEX_EXCLUSIVE;
      if (c[kFitUncordoned] > 0u) flags |= LWSE_PEX_CORDONED;
      if (!pinned && q.size < 1) flags |= LWSE_PEX_BAD_SIZE;
      if (pinned) {
        uint32_t ld = LWSE_NONE;
        if (q.leader_node < p.n_nodes) {
          const uint4 nr = __ldg(reinterpret_cast<const uint4*>(p.nodes + q.leader_node));
          if (((nr.w >> 16) & LWSE_NODE_HAS_TOPOLOGY) && nr.z < p.n_domains) ld = nr.z;
        }
        if (ld == LWSE_NONE) {
          flags |= LWSE_PEX_NO_CLAIM;
        } else {
          const unsigned long long hk = explain_holder(p, q.ns, ld);
          if (hk != kExplainEmpty && hk < key && !(hk >> 63)) {
            flags |= LWSE_PEX_CONFLICT;
            blk_d = ld;
            blk_row = (uint32_t)(hk & 0xFFFFFFu);
          }
        }
      }
    }
    if (lane == 0) {
      if (k < p.capacity) {
        uint4* o = reinterpret_cast<uint4*>(p.out + k);
        o[0] = make_uint4(r, flags, place_flags, c[kOwn]);
        o[1] = make_uint4(c[kNoUsable], c[kTooSmall], c[kHeldPinned], c[kHeldEarlier]);
        o[2] = make_uint4(c[kHeldLater], c[kOpen], c[kFitUncordoned], best_d);
        o[3] = make_uint4(blk_d, blk_row, short_v, short_d);
      }
      for (uint32_t j = 0; j < kFit; j++)
        if (c[j]) atomicAdd(p.totals + j, (unsigned long long)c[j]);
      for (uint32_t b = 0; b < 7u; b++)
        if (flags & (1u << b)) atomicAdd(p.totals + 8u + b, 1ull);
    }
  }
}

int launch_place_explain(const PlaceExplainLaunch* p, int sm_count, cudaStream_t s) {
  const uint32_t cap = (uint32_t)sm_count * 8u;
  place_explain_stats_kernel<<<grid_for(p->n_nodes, 256, cap), 256, 0, s>>>(*p);
  int kernels = 1;
  if (p->by_mask) {
    const uint32_t n_chunks = (p->n_rows + kExplainChunk - 1u) / kExplainChunk;
    place_explain_count_kernel<<<grid_for(n_chunks, 1, cap), kExplainChunk, 0, s>>>(*p);
    if (const int r = launch_result(0); r < 0) return r;
    if (const int r = launch_index_scan(p->chunk_count, p->chunk_first, p->chunk_cursor, n_chunks, s); r < 0) return r;
    place_explain_fill_kernel<<<grid_for(n_chunks, 1, cap), kExplainChunk, 0, s>>>(*p);
    kernels += 3;
  } else {
    place_explain_mark_kernel<<<grid_for(p->n_listed, 256, cap), 256, 0, s>>>(*p);
    kernels += 1;
  }
  place_explain_hold_kernel<<<grid_for(p->n_rows, 256, cap), 256, 0, s>>>(*p);
  place_explain_kernel<<<grid_for(p->n_listed, 8, cap), 256, 0, s>>>(*p);
  return launch_result(kernels + 2);
}

}  // namespace lwse
