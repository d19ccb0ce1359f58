// The LWS-level pass of one LeaderWorkerSet (sm_90a): the status counters, the conditions and
// rollingUpdateParameters with the partition walk, over the object's flag bytes.  Shared by
// lws_sweep_kernel (lwse_lws_kernels.cu) and the rollout forecast (lwse_lws_forecast_kernels.cu),
// so that the forecast replays the sweep's own arithmetic.
#pragma once

#include "lwse_device.cuh"

namespace lwse {

__device__ __forceinline__ int32_t want_replicas(int32_t lws_replicas, int32_t surge, int32_t mu,
                                                 int32_t unready, int32_t sts_replicas,
                                                 uint32_t& event) {
  // calculateRollingUpdateReplicas :685-696
  int32_t fin;
  if (unready <= surge) {
    fin = lws_replicas + max(0, unready - mu);
  } else {
    fin = lws_replicas + surge;
  }
  if (fin == sts_replicas - 1)  // :313
    event = LWSE_EVENT_DELETE_ONE;
  else if (fin < sts_replicas)  // :315
    event = LWSE_EVENT_DELETE_RANGE;
  return fin;
}

// Byte-lane masks of one 64-bit word of the flag column.  Byte b of word j is group slot
// idx = off + b of the object (off = 8 j - group_base, negative in the object's first word).
constexpr uint64_t kLaneOnes = 0x0101010101010101ull;
__device__ __forceinline__ uint64_t lanes_upto(int64_t n) {  // bit 0 of bytes [0, n)
  if (n <= 0) return 0ull;
  if (n >= 8) return kLaneOnes;
  return kLaneOnes & ((1ull << (8 * (int)n)) - 1ull);
}
__device__ __forceinline__ uint64_t lanes_idx_range(int32_t off, int32_t lo, int32_t hi) {  // lo <= idx < hi
  return lanes_upto((int64_t)hi - off) & ~lanes_upto((int64_t)lo - off);
}
__device__ __forceinline__ int32_t highest_lane(uint64_t m) { return (63 - __clzll((long long)m)) >> 3; }  // m != 0

// How the pass loads a word of flag bytes.  The sweep reads the column the group pass wrote in an
// earlier kernel (ld.global.cg); the forecast reads its private copy, which the tile rewrites between
// passes (plain coherent loads, ordered by __syncwarp).
struct FlagLoadCg {
  __device__ __forceinline__ uint64_t operator()(const uint64_t* p) const { return __ldcg(p); }
};
struct FlagLoadCoherent {
  __device__ __forceinline__ uint64_t operator()(const uint64_t* p) const { return *p; }
};

// One object's lwse_lws_out row as two 16-byte words.
struct LwsPassOut {
  uint4 v0;  // {sts_partition, sts_replicas, sts_max_unavailable, ready_replicas}
  uint4 v1;  // {updated_replicas, min_member, flags, unready_replicas}
};

// The pass of one object whose 64-byte row is r0..r3, over the flag bytes of group rows
// [group_base, group_base + group_count) of `words` (a column of n_groups bytes, padded to 8).  All W
// lanes of the tile call it with the same row and get the same result.
template <int W, class Ld>
__device__ __forceinline__ LwsPassOut lws_pass_one(const uint4 r0, const uint4 r1, const uint4 r2, const uint4 r3,
                                                   const uint64_t* words, const uint32_t n_groups,
                                                   const uint32_t sweep_flags, const uint32_t lane) {
  const Ld ld{};
  const int32_t size = (int32_t)r0.z;
  const uint32_t lflags = r0.w;
  const int32_t R = (int32_t)r1.x, P = (int32_t)r1.y;
  const int32_t n = (int32_t)r2.x;  // sts replicas
  const int32_t cur_partition = (int32_t)r2.y, annot = (int32_t)r2.z;
  const uint32_t gbase = r3.z, gc = r3.w;

  uint32_t oflags = 0, event = LWSE_EVENT_NONE;
  int32_t o_partition = 0, o_replicas = 0, o_mu = 0, o_ready = 0, o_updated = 0, o_unready = 0,
          o_min_member = 0;

  if ((uint64_t)gbase + gc > n_groups) {
    oflags = LWSE_LOUT_BAD_TABLE;
  } else {
    const bool sts_exists = lflags & LWSE_LWS_STS_EXISTS;
    const bool intstr_bad = lflags & LWSE_LWS_INTSTR_INVALID;
    int32_t mu = scaled_value((int32_t)r1.w, lflags & LWSE_LWS_UNAVAIL_IS_PERCENT, R, false);
    int32_t surge = scaled_value((int32_t)r1.z, lflags & LWSE_LWS_SURGE_IS_PERCENT, R, true);
    if (surge > R) surge = R;  // :307
    const int32_t burst = R + surge;
    const int32_t gcs = (int32_t)min(gc, 0x7FFFFFFFu);
    const uint32_t j0 = gbase >> 3, j1 = gc ? ((gbase + gc - 1u) >> 3) : j0;  // words of the object's flag bytes

    // ---- pass A: counters over every group slot of the object ----
    // updateConditions counters (:450-475) and, for slots below the leader
    // sts's replica count, the getReplicaStates view.
    int32_t c_ready = 0, c_updated = 0, c_cur_nb = 0, c_upd_nb = 0, c_ready_nb = 0, c_upd_rdy = 0;
    int32_t c_ok_below_R = 0;  // slots < min(R, n) that are ready ∧ updated
    int32_t max_bad = -1;      // highest slot < n that is not (ready ∧ updated)
    const int32_t n_live = min(n, gcs);
    if (gc) {
      for (uint32_t j = j0 + lane; j <= j1; j += W) {
        const uint64_t w = ld(words + j);
        const int32_t off = (int32_t)(j << 3) - (int32_t)gbase;  // |off| < 2^31: n_groups < 2^31 in practice
        const uint64_t valid = lanes_idx_range(off, 0, gcs);
        const uint64_t st_rd = w & kLaneOnes, st_up = (w >> 1) & kLaneOnes;
        const uint64_t cnt = (w >> 2) & valid, rd = (w >> 3) & kLaneOnes, up = (w >> 4) & kLaneOnes;
        const uint64_t in_R = lanes_idx_range(off, 0, R), in_nb = lanes_idx_range(off, P, R);
        c_ready += __popcll(cnt & rd);
        c_updated += __popcll(cnt & up);
        c_cur_nb += __popcll(cnt & in_nb);
        c_upd_nb += __popcll(cnt & in_nb & up);
        c_ready_nb += __popcll(cnt & in_R & rd);
        c_upd_rdy += __popcll(cnt & in_nb & rd & up);
        const uint64_t live = valid & lanes_idx_range(off, 0, n_live), ok = st_rd & st_up;
        c_ok_below_R += __popcll(ok & live & in_R);
        const uint64_t badm = live & ~ok;
        if (badm) max_bad = off + highest_lane(badm);  // j ascends per lane
      }
    }
    c_ready = tile_add<W>(c_ready);
    c_updated = tile_add<W>(c_updated);
    c_cur_nb = tile_add<W>(c_cur_nb);
    c_upd_nb = tile_add<W>(c_upd_nb);
    c_ready_nb = tile_add<W>(c_ready_nb);
    c_upd_rdy = tile_add<W>(c_upd_rdy);
    c_ok_below_R = tile_add<W>(c_ok_below_R);
    max_bad = tile_max<W>(max_bad);
    if (n > n_live) max_bad = n - 1;  // slots without any object are zero-valued states

    // ---- status / conditions (:478-501) ----
    if (lflags & LWSE_LWS_GROUP_LABEL_INVALID) {
      oflags |= LWSE_LOUT_STATUS_ERROR;  // :434-437
    } else {
      o_ready = c_ready;
      o_updated = c_updated;
      uint32_t cond;
      if (c_upd_nb < c_cur_nb)
        cond = LWSE_COND_UPDATE_IN_PROGRESS;
      else if (c_ready_nb == R && c_upd_rdy == c_cur_nb)
        cond = LWSE_COND_AVAILABLE;
      else
        cond = LWSE_COND_PROGRESSING;
      oflags |= cond << LWSE_LOUT_COND_SHIFT;
      if (P == 0 && c_upd_rdy == R) oflags |= LWSE_LOUT_UPDATE_DONE;
    }

    // ---- rollingUpdateParameters (:280-373) ----
    bool err = false;
    if (!sts_exists) {  // Case 1
      o_partition = 0;
      o_replicas = R;
    } else if (intstr_bad) {
      err = true;
    } else if (lflags & LWSE_LWS_UPDATED) {  // Case 2
      o_partition = min(R, n);
      o_replicas = n < R ? R : want_replicas(R, surge, mu, R, n, event);
    } else if (cur_partition == 0 && n == R) {  // Case 3
      o_partition = 0;
      o_replicas = R;
    } else if (n < R) {
      o_partition = cur_partition;
      o_replicas = R;
    } else {
      // calculateLWSUnreadyReplicas :675-683 (R >= 0 here because n >= R is not implied; clamp)
      const int32_t unready = max(R, 0) - c_ok_below_R;
      o_unready = unready;
      if (!(lflags & LWSE_LWS_ANNOT_VALID)) {
        err = true;  // :351-354
      } else if (annot != R) {  // Case 4
        o_partition = min(cur_partition, burst);
        o_replicas = want_replicas(R, surge, mu, unready, n, event);
      } else {  // Case 5
        const int32_t step = mu + surge - (burst - n);  // :366-369
        // rollingUpdatePartition :643-673
        const int32_t cont_ready = n - 1 - max_bad;  // calculateContinuousReadyReplicas
        const int32_t rsp = max(0, n - cont_ready - step);
        // pass B: unavailable = #{idx < rsp : !ready}
        int32_t unavail = 0;
        const int32_t rsp_live = min(rsp, n_live);
        if (rsp_live > 0) {
          const uint32_t jb = (gbase + (uint32_t)rsp_live - 1u) >> 3;
          for (uint32_t j = j0 + lane; j <= jb; j += W) {
            const int32_t off = (int32_t)(j << 3) - (int32_t)gbase;
            unavail += __popcll(~ld(words + j) & lanes_idx_range(off, 0, rsp_live));
          }
        }
        unavail = tile_add<W>(unavail) + (rsp - rsp_live);
        int32_t part = rsp + unavail;
        const int32_t hi = min(part, n - 1);
        if (hi >= rsp) {
          // pass C: the walk stops at the highest idx in [rsp, hi] that is ready ∧ ¬updated
          int32_t blocker = -1;
          const int32_t hi_live = min(hi, n_live - 1);
          if (hi_live >= rsp) {
            const uint32_t ja = (gbase + (uint32_t)rsp) >> 3, jb = (gbase + (uint32_t)hi_live) >> 3;
            for (uint32_t j = ja + lane; j <= jb; j += W) {
              const uint64_t w = ld(words + j);
              const int32_t off = (int32_t)(j << 3) - (int32_t)gbase;
              const uint64_t m = w & ~(w >> 1) & lanes_idx_range(off, rsp, hi_live + 1);
              if (m) blocker = off + highest_lane(m);
            }
          }
          blocker = tile_max<W>(blocker);
          if (blocker < 0)
            part = rsp;
          else if (blocker < hi)
            part = blocker + 1;
          // blocker == hi: the first probe breaks, partition keeps rsp + unavail
        }
        o_partition = min(part, cur_partition);
        o_replicas = want_replicas(R, surge, mu, unready, n, event);
      }
    }
    if (err) {
      oflags |= LWSE_LOUT_RUP_ERROR;
      o_partition = 0;
      o_replicas = 0;
      event = LWSE_EVENT_NONE;
    }
    o_partition = max(o_partition, P);  // deferred clamp :285-288
    oflags |= event << LWSE_LOUT_EVENT_SHIFT;

    // stsMaxUnavailable :811-830
    if (!intstr_bad) o_mu = max(1, mu + surge);
    // PodGroup MinMember, volcano_provider.go:72,81-83
    if (sweep_flags & LWSE_SWEEP_GANG) o_min_member = (lflags & LWSE_LWS_STARTUP_LEADER_READY) ? 1 : size;
    if (lflags & LWSE_LWS_IRREGULAR) oflags |= LWSE_LOUT_IRREGULAR;
  }
  return LwsPassOut{make_uint4((uint32_t)o_partition, (uint32_t)o_replicas, (uint32_t)o_mu, (uint32_t)o_ready),
                    make_uint4((uint32_t)o_updated, (uint32_t)o_min_member, oflags, (uint32_t)o_unready)};
}

}  // namespace lwse
