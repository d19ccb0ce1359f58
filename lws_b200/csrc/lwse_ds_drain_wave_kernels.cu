// DS drain waves (lwse_resident_ds_drain_waves, sm_90a); the definition is in lwse.h, the argument in DESIGN.md §3.5.
//
// Around the drain waves chain (lwse_drain_wave_kernels.cu), after the before sweep of the DS drain:
//   ds_drain_waves_caps_kernel    one thread per DS: every revision-role row its sweep reads that takes an LWS value
//                                 (the link rule) ORs kCapLinked into caps[L], and the verdict bit of the DS's flags
//                                 in the before sweep that gates it: DS_SERVICE (a new-revision spec row of a
//                                 NEW_READY DS), DS_OLD_SERVICE (a spec row of old revision v with bit v of
//                                 ready_revs), DS_STALL (a new-revision spec row of a STABLE DS).  BAD_TABLE DS and
//                                 removed roles add no verdict bit.
//   (launch_drain_waves_capped: the pairs bound by evaluated or linked rows, the dense rows' slacks, the plan.)
//   ds_drain_waves_finish_kernel  the answer: per DS, over its linked rows, lost(dense L, w) of every wave into the
//                                 wave's rows touched / zeroed and its DS verdicts (each gated as in the per-key
//                                 form); per evaluated dense row, the waves in which it falls below its floor; per key
//                                 the plan's status and the alone columns of both per-key forms; per wave the plan's
//                                 LWS columns.  The DS and breach columns are summed with atomics into words no other
//                                 thread stores to.
#include "lwse_device.cuh"
#include "lwse_launch.cuh"

namespace lwse {

__global__ void __launch_bounds__(128) ds_drain_waves_caps_kernel(const DsDrainWavesLaunch d) {
  const lwse_ds_tables& t = d.t;
  for (uint32_t ds = blockIdx.x * blockDim.x + threadIdx.x; ds < t.n_ds; ds += gridDim.x * blockDim.x) {
    const uint4 h0 = ldg_stream(reinterpret_cast<const uint4*>(t.ds + ds) + 0);
    const uint4 h1 = ldg_stream(reinterpret_cast<const uint4*>(t.ds + ds) + 1);
    if (!ds_rows_ok(t, h0, h1)) continue;  // BAD_TABLE
    const uint4 before = __ldcg(reinterpret_cast<const uint4*>(t.ds_out + ds));  // {flags, drained_revs, ready_revs, 0}
    const uint32_t n = h0.w, S = h1.x, rev_base = h1.y, V = h1.z;
    for (uint32_t r = 0; r <= V; r++)
      for (uint32_t i = 0; i < n; i++) {
        const uint32_t row = rev_base + r * n + i;
        const uint32_t L = ds_link_target(d.lk.links, d.lk.lws, d.lk.lws_out, d.lk.n_lws, row,
                                          __ldg(&t.revroles[row].flags) & LWSE_RR_EXISTS);
        if (L == LWSE_NONE) continue;
        uint32_t bits = kCapLinked;
        if (i < S) {
          if (r == V) {
            if (before.x & LWSE_DOUT_NEW_READY) bits |= LWSE_DSW_DS_SERVICE;
            if (before.x & LWSE_DOUT_STABLE) bits |= LWSE_DSW_DS_STALL;
          } else if ((before.z >> r) & 1u) {
            bits |= LWSE_DSW_DS_OLD_SERVICE;
          }
        }
        atomicOr(d.caps + L, bits);
      }
  }
}

__device__ __forceinline__ uint32_t* wave_words(const DsDrainWavesLaunch& d, uint32_t m, uint32_t w) {
  return reinterpret_cast<uint32_t*>(d.out + 16 + (size_t)m * sizeof(lwse_ds_drain_wave_key) + (size_t)w * sizeof(lwse_ds_drain_wave));
}

// Word offsets in lwse_ds_drain_wave.
constexpr uint32_t kWvLwsBreached = 2, kWvDsTouched = 9, kWvService = 10, kWvOldService = 11, kWvStalled = 12,
                   kWvRowsTouched = 13, kWvRowsZeroed = 14;

__global__ void __launch_bounds__(256) ds_drain_waves_finish_kernel(const DsDrainWavesLaunch d, const DrainWavesLaunch w) {
  const uint32_t n_open = __ldcg(reinterpret_cast<const uint32_t*>(w.out));
  const uint8_t* plan_waves = w.out + 16 + (size_t)w.m * sizeof(lwse_drain_wave_key);
  const lwse_ds_tables& t = d.t;
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t n = max(max(t.n_ds, w.n_dense), max(w.m, n_open));
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (i < t.n_ds && n_open) {
      const uint4 h0 = ldg_stream(reinterpret_cast<const uint4*>(t.ds + i) + 0);
      const uint4 h1 = ldg_stream(reinterpret_cast<const uint4*>(t.ds + i) + 1);
      if (ds_rows_ok(t, h0, h1)) {
        const uint4 before = __ldcg(reinterpret_cast<const uint4*>(t.ds_out + i));
        const uint32_t nr = h0.w, S = h1.x, rev_base = h1.y, V = h1.z, nrr = (V + 1u) * nr;
        unsigned long long touched = 0, new_zeroed = 0, new_changed = 0, old_fell = 0;
        for (uint32_t k = 0; k < nrr; k++) {
          const uint32_t row = rev_base + k;
          const uint32_t L = ds_link_target(d.lk.links, d.lk.lws, d.lk.lws_out, d.lk.n_lws, row,
                                            __ldg(&t.revroles[row].flags) & LWSE_RR_EXISTS);
          if (L == LWSE_NONE) continue;
          const uint32_t dl = __ldcg(w.l_first + L);
          if (__ldcg(w.l_first + L + 1) == dl) continue;  // no restarted member group of L in any key
          const int32_t rb = __ldg(&d.lk.lws_out[L].ready_replicas);
          const uint32_t r = k / nr, role = k - r * nr;
          unsigned long long ws = __ldcg(w.row_waves + 2u * dl);
          while (ws) {
            const uint32_t v = (uint32_t)(__ffsll((long long)ws) - 1);
            ws &= ws - 1ull;
            const uint32_t lost = __ldcg(w.lost + (size_t)dl * w.cols + v);
            if (lost == 0) continue;
            const unsigned long long bit = 1ull << v;
            const int32_t ra = clamp_i32((int64_t)rb - lost);
            const bool zero = rb >= 1 && ra < 1;
            touched |= bit;
            uint32_t* row_w = wave_words(d, w.m, v);
            atomicAdd(row_w + kWvRowsTouched, 1u);
            if (zero) atomicAdd(row_w + kWvRowsZeroed, 1u);
            if (role >= S) continue;  // (a removed role serves nothing)
            if (r == V) {
              if (zero) new_zeroed |= bit;
              if (ra != rb) new_changed |= bit;
            } else if (zero && ((before.z >> r) & 1u)) {
              old_fell |= bit;
            }
          }
        }
        while (touched) {
          const uint32_t v = (uint32_t)(__ffsll((long long)touched) - 1);
          const unsigned long long bit = 1ull << v;
          touched &= touched - 1ull;
          uint32_t* row_w = wave_words(d, w.m, v);
          atomicAdd(row_w + kWvDsTouched, 1u);
          if ((new_zeroed & bit) && (before.x & LWSE_DOUT_NEW_READY)) atomicAdd(row_w + kWvService, 1u);
          if (old_fell & bit) atomicAdd(row_w + kWvOldService, 1u);
          if ((new_changed & bit) && (before.x & LWSE_DOUT_STABLE)) atomicAdd(row_w + kWvStalled, 1u);
        }
      }
    }
    if (i < w.n_dense) {
      const uint4 dr = __ldg(w.dense + i);  // {ready_before, floor, flags, slack}
      if (dr.z & 1u) {                      // (kDenseEvaluated)
        unsigned long long ws = __ldcg(w.row_waves + 2u * i);
        while (ws) {
          const uint32_t v = (uint32_t)(__ffsll((long long)ws) - 1);
          ws &= ws - 1ull;
          const uint32_t lost = __ldcg(w.lost + (size_t)i * w.cols + v);
          if (lost > 0 && (int64_t)(int32_t)dr.x - lost < (int64_t)(int32_t)dr.y)
            atomicAdd(wave_words(d, w.m, v) + kWvLwsBreached, 1u);
        }
      }
    }
    if (i < w.m) {
      const uint4 k0 = __ldcg(reinterpret_cast<const uint4*>(w.out + 16 + (size_t)i * sizeof(lwse_drain_wave_key)));
      const lwse_drain_budget_cost* c = w.cost + k0.x;
      const uint4 dc = __ldg(reinterpret_cast<const uint4*>(d.ds_cost + k0.x));  // {touched, service, old, stalled}
      const uint32_t breached = __ldg(&c->lws_breached);
      const uint32_t alone = (breached ? LWSE_DSW_LWS_FLOOR : 0u) | (dc.y ? LWSE_DSW_DS_SERVICE : 0u) |
                             (dc.z ? LWSE_DSW_DS_OLD_SERVICE : 0u) | (dc.w ? LWSE_DSW_DS_STALL : 0u);
      uint4* row = reinterpret_cast<uint4*>(d.out + 16 + (size_t)i * sizeof(lwse_ds_drain_wave_key));
      row[0] = make_uint4(k0.x, k0.y, k0.z, alone);
      row[1] = make_uint4(__ldg(&c->groups_restarted), __ldg(&c->ready_restarted), __ldg(&c->lws_touched), breached);
      row[2] = dc;
    }
    if (i < n_open) {
      const lwse_drain_wave* src = reinterpret_cast<const lwse_drain_wave*>(plan_waves) + i;
      lwse_ds_drain_wave* dst = reinterpret_cast<lwse_ds_drain_wave*>(wave_words(d, w.m, i));
      dst->n_keys = __ldcg(&src->n_keys);
      dst->lws_touched = __ldcg(&src->lws_touched);
      dst->lws_loses_available = __ldcg(&src->lws_loses_available);
      dst->n_pods_evicted = __ldcg(&src->n_pods_evicted);
      dst->n_leaders_evicted = __ldcg(&src->n_leaders_evicted);
      dst->n_groups_restarted = __ldcg(&src->n_groups_restarted);
      dst->n_ready_restarted = __ldcg(&src->n_ready_restarted);
      dst->min_margin = __ldcg(&src->min_margin);
      dst->n_pods_recreated = __ldcg(reinterpret_cast<const unsigned long long*>(&src->n_pods_recreated));
    }
    if (i == 0) *reinterpret_cast<uint4*>(d.out) = __ldcg(reinterpret_cast<const uint4*>(w.out));
  }
}

int launch_ds_drain_waves(const DsDrainWavesLaunch* d, const DrainWavesLaunch* w, int pass, int sm_count, cudaStream_t s) {
  if (pass == 0) {
    if (d->t.n_ds == 0) return 0;
    ds_drain_waves_caps_kernel<<<grid_for(d->t.n_ds, 128, (uint32_t)sm_count * 16u), 128, 0, s>>>(*d);
    return launch_result(1);
  }
  uint32_t n = d->t.n_ds > w->n_dense ? d->t.n_ds : w->n_dense;
  n = n > w->m ? n : w->m;
  n = n > d->max_waves ? n : d->max_waves;
  ds_drain_waves_finish_kernel<<<grid_for(n, 256, (uint32_t)sm_count * 4u), 256, 0, s>>>(*d, *w);
  return launch_result(1);
}

}  // namespace lwse
