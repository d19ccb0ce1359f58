// DS rollout what-if (lwse_resident_ds_rollout_whatif, sm_90a); the definition is in lwse.h.
//
//   ds_whatif_count_kernel    one thread per proposal: BAD_TABLE or V' from the resident DS row, and the
//                             revision-role rows it gathers, (V' + 1) * n
//   scan (three kernels)      the counts → each proposal's first scratch row, and the total (lwse_device.cuh)
//   ds_whatif_gather_kernel   one warp per proposal: scratch DS row i, its role rows at 10 * i, and its
//                             revision-role and link rows, the retired revision's absent new rows last
// The engine then runs the linked DS sweep (`now`) and the DS forecast over the scratch tables.
#include "lwse_device.cuh"
#include "lwse_launch.cuh"

namespace lwse {

// V' of a proposal with flags `pflags` on the resident DS row (h0, h1), or LWSE_NONE when it is BAD_TABLE: the
// resident row fails the table checks, or retiring its target revision takes it past LWSE_DS_MAX_OLD_REVS.
__device__ __forceinline__ uint32_t ds_whatif_old_revs(const lwse_ds_tables& t, const uint4 h0, const uint4 h1,
                                                       const uint32_t pflags) {
  if (!ds_rows_ok(t, h0, h1)) return LWSE_NONE;
  const bool retire = (pflags & LWSE_DSP_NEW_REVISION) && (h1.w & LWSE_DS_HAS_NEW_REVISION);
  const uint32_t v = h1.z + (retire ? 1u : 0u);
  return v > LWSE_DS_MAX_OLD_REVS ? LWSE_NONE : v;
}

__global__ void __launch_bounds__(256) ds_whatif_count_kernel(const DsWhatifHost a) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
    const uint2 p = __ldg(reinterpret_cast<const uint2*>(a.proposals) + i);  // {ds, flags}
    const uint4 h0 = ldg_stream(reinterpret_cast<const uint4*>(a.t.ds + p.x) + 0);
    const uint4 h1 = ldg_stream(reinterpret_cast<const uint4*>(a.t.ds + p.x) + 1);
    const uint32_t v = ds_whatif_old_revs(a.t, h0, h1, p.y);
    a.count[i] = v == LWSE_NONE ? 0u : (v + 1u) * h0.w;  // <= 33 * 10
  }
}

// The layout: the counts → exclusive offsets (launch_forecast_scan).
struct DsWhatifLayoutOp {
  const uint32_t* rows;
  uint32_t* off;
  __device__ __forceinline__ unsigned long long count(uint32_t i) const { return __ldg(rows + i); }
  __device__ __forceinline__ unsigned long long apply(uint32_t i, unsigned long long base, unsigned long long) const {
    off[i] = (uint32_t)base;  // < 2^32: n <= LWSE_DS_WHATIF_MAX_PROPOSALS rows of at most 330
    return 0ull;
  }
};

__global__ void __launch_bounds__(256) ds_whatif_gather_kernel(const DsWhatifHost a) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t n_warps = gridDim.x * (blockDim.x >> 5);
  for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < a.n; i += n_warps) {
    const uint2 p = __ldg(reinterpret_cast<const uint2*>(a.proposals) + i);
    const uint4 h0 = ldg_stream(reinterpret_cast<const uint4*>(a.t.ds + p.x) + 0);
    const uint4 h1 = ldg_stream(reinterpret_cast<const uint4*>(a.t.ds + p.x) + 1);
    const uint32_t v = ds_whatif_old_revs(a.t, h0, h1, p.y);
    const bool bad = v == LWSE_NONE;
    const uint32_t n = h0.w, base = __ldg(a.off + i);
    if (lane == 0) {
      // a BAD proposal's rev_base is LWSE_NONE, beyond any scratch table (the 64-bit range test of
      // ds_rows_ok), so that the sweep and the forecast report it BAD_TABLE and read none of its rows
      uint4* w = reinterpret_cast<uint4*>(a.s_ds + i);
      w[0] = make_uint4(h0.x, h0.y, i * LWSE_DS_MAX_ROLES, n);
      const uint32_t flags = (!bad && v != h1.z) ? (h1.w & ~LWSE_DS_HAS_NEW_REVISION) : h1.w;
      w[1] = make_uint4(h1.x, bad ? LWSE_NONE : base, bad ? h1.z : v, flags);
    }
    if (bad) continue;
    if (lane < n) {
      const uint4 r = (p.y & LWSE_DSP_ROLES) ? ldg_stream(a.q_roles + (size_t)i * LWSE_DS_MAX_ROLES + lane)
                                             : ldg_stream(a.t.roles + h0.z + lane);
      reinterpret_cast<uint4*>(a.s_roles)[(size_t)i * LWSE_DS_MAX_ROLES + lane] = r;
    }
    // rows [0, (V + 1) n) as resident (the retired target revision is old revision V), then, when it
    // retires, n absent rows of the new revision that carry no link
    const uint32_t n_copy = (h1.z + 1u) * n, n_rows = (v + 1u) * n;
    const uint4* src = reinterpret_cast<const uint4*>(a.t.revroles + h1.y);
    const uint4* lsrc = reinterpret_cast<const uint4*>(a.links + h1.y);
    uint4* dst = reinterpret_cast<uint4*>(a.s_revroles + base);
    uint4* ldst = reinterpret_cast<uint4*>(a.s_links + base);
    for (uint32_t k = lane; k < n_rows; k += 32u) {
      const bool copy = k < n_copy;
      dst[k] = copy ? ldg_stream(src + k) : make_uint4(0u, 0xFFFFFFFFu, 0u, 0u);  // {0, -1, 0, 0}
      ldst[k] = copy ? ldg_stream(lsrc + k) : make_uint4(0u, 0u, LWSE_NONE, 0u);
    }
  }
}

int launch_ds_whatif_layout(const DsWhatifHost* h, unsigned long long* sums, unsigned long long* total, int sm_count,
                            cudaStream_t s) {
  int launched = 0;
  if (h->n) {
    const uint32_t want = (h->n + 255u) / 256u, cap = (uint32_t)sm_count * 8u;
    ds_whatif_count_kernel<<<want < cap ? want : cap, 256, 0, s>>>(*h);
    launched = 1;
  }
  launch_forecast_scan(DsWhatifLayoutOp{h->count, h->off}, h->n, sums, total, nullptr, s);
  return launch_result(launched + (h->n ? 3 : 1));
}

int launch_ds_whatif_gather(const DsWhatifHost* h, int sm_count, cudaStream_t s) {
  if (h->n == 0) return 0;
  const uint32_t want = (h->n + 7u) / 8u, cap = (uint32_t)sm_count * 8u;
  ds_whatif_gather_kernel<<<want < cap ? want : cap, 256, 0, s>>>(*h);
  return launch_result(1);
}

}  // namespace lwse
