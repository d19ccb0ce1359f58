// Rolling-update forecast of LeaderWorkerSets (lwse_lws_forecast_*, sm_90a); the model is in lwse.h.
//
//   lws_forecast_slots_kernel      C (rounded up to 8) private flag slots per object
//   scan (three kernels)           their exclusive prefix, and the total (lwse_device.cuh)
//   lws_forecast_kernel<W, false>  one W-lane tile per object: copies its flag bytes into its private
//                                  slots and replays its cycles through lws_pass_one (the sweep's
//                                  own pass); summaries, and its trajectory row count
//   scan (three kernels)           trajectory offsets, TRUNCATED (lwse_device.cuh)
//   lws_forecast_kernel<W, true>   the replay again, writing the rows the scan reserved
#include "lwse_device.cuh"
#include "lwse_launch.cuh"
#include "lwse_lws_pass.cuh"

namespace lwse {

struct LwsForecastArgs {
  const lwse_lws_rec* lws;
  uint32_t n_lws;
  const lwse_group_out* group_out;  // the group results the forecast starts from
  uint32_t n_groups;
  const unsigned long long* slot_off;  // [n_lws] first private slot of each object (a multiple of 8)
  uint8_t* slots;                      // private flag bytes
  uint32_t n_slots;                    // < 2^31
  lwse_lws_forecast* fc;               // [n_lws]
  lwse_lws_forecast_step* steps;       // [steps_rows] (write pass only)
  uint32_t steps_rows;                 // rows of `steps`: those the scan counted as written
  unsigned long long* refused;         // += accesses the bounds checks below refused (0 unless the layout is wrong)
};

constexpr uint32_t kForecastFlagMask = LWSE_GOUT_STATE_READY | LWSE_GOUT_STATE_UPDATED | LWSE_GOUT_COUNTED |
                                       LWSE_GOUT_COND_READY | LWSE_GOUT_COND_UPDATED;
static_assert(kForecastFlagMask == 0x1Fu, "flag bytes are the low five bits of group_out.flags");

// C of an object (lwse.h), or -1 when its group range is outside the group table.
__device__ __forceinline__ long long forecast_slots_of(const uint4 r0, const uint4 r1, const uint4 r2, const uint4 r3,
                                                       uint32_t n_groups) {
  const uint32_t gbase = r3.z, gc = r3.w;
  if ((uint64_t)gbase + gc > n_groups) return -1;
  const int32_t R = (int32_t)r1.x;
  int32_t surge = scaled_value((int32_t)r1.z, r0.w & LWSE_LWS_SURGE_IS_PERCENT, R, true);
  surge = max(min(surge, R), 0);
  const long long want = max((long long)(int32_t)r2.x, (long long)R + surge);
  return max((long long)gc, max(want, 0ll));
}

__global__ void __launch_bounds__(256) lws_forecast_slots_kernel(const LwsForecastArgs a,
                                                                 unsigned long long* counts) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n_lws; i += gridDim.x * blockDim.x) {
    const uint4* row = reinterpret_cast<const uint4*>(a.lws + i);
    const long long C = forecast_slots_of(ldg_stream(row), ldg_stream(row + 1), ldg_stream(row + 2),
                                          ldg_stream(row + 3), a.n_groups);
    counts[i] = (C < 0 || C > (long long)LWSE_LWS_FORECAST_MAX_SLOTS) ? 0ull : (unsigned long long)((C + 7) & ~7ll);
  }
}

// The slot layout: counts → exclusive offsets in place (launch_forecast_scan).
struct SlotLayoutOp {
  unsigned long long* v;
  __device__ __forceinline__ unsigned long long count(uint32_t i) const { return v[i]; }
  __device__ __forceinline__ unsigned long long apply(uint32_t i, unsigned long long base, unsigned long long) const {
    v[i] = base;
    return 0ull;
  }
};

template <int W>
__device__ __forceinline__ void tile_sync() {
  if constexpr (W > 1) __syncwarp(tile_mask<W>());
}

// The replay of object i by one W-lane tile.  kWrite = false: the summary, with the object's row count
// in step_base (the scan turns it into an offset).  kWrite = true: replays the object again and writes
// at most the rows the scan reserved for it.  The tile owns the object's private slots.
template <int W, bool kWrite>
__device__ __forceinline__ void lws_forecast_one(const LwsForecastArgs& a, const uint32_t i, const uint32_t lane) {
  const uint4* row = reinterpret_cast<const uint4*>(a.lws + i);
  const uint4 r0 = ldg_stream(row + 0), r1 = ldg_stream(row + 1);
  uint4 r2 = ldg_stream(row + 2), r3 = ldg_stream(row + 3);
  const long long C = forecast_slots_of(r0, r1, r2, r3, a.n_groups);
  if (C < 0 || C > (long long)LWSE_LWS_FORECAST_MAX_SLOTS) {
    if (!kWrite && lane == 0)
      a.fc[i] = lwse_lws_forecast{C < 0 ? LWSE_LWSF_BAD_TABLE : LWSE_LWSF_NOT_FORECAST, 0u, 0u, 0u, 0, 0, 0, 0};
    return;
  }
  uint32_t step_base = 0, step_limit = 0;
  if constexpr (kWrite) {
    const lwse_lws_forecast c = a.fc[i];
    if (c.n_steps == 0 || (c.flags & LWSE_LWSF_TRUNCATED)) return;
    step_base = c.step_base;
    step_limit = c.n_steps;
  }
  // the private slots [base, base + C8): the object's flag bytes, then zeros
  const uint32_t gbase = r3.z, gc = r3.w;
  const uint32_t base = (uint32_t)a.slot_off[i], n_words = (uint32_t)((C + 7) >> 3);
  // Every slot the object's tile touches (the copy, the apply, and the pass's reads of words
  // [base / 8, (base + C - 1) / 8]) lies in [base, base + 8 * n_words); refuse the object if that range is
  // not inside the scratch the slot scan sized.
  if ((unsigned long long)base + 8ull * n_words > a.n_slots) {
    if (lane == 0) atomicAdd(a.refused, 1ull);
    return;
  }
  uint64_t* words = reinterpret_cast<uint64_t*>(a.slots + base);
  for (uint32_t k = lane; k < n_words; k += W) {
    uint64_t w = 0;
    for (uint32_t b = 0; b < 8u; b++) {
      const uint32_t idx = 8u * k + b;
      if (idx < gc) w |= (uint64_t)(__ldg(&a.group_out[gbase + idx].flags) & kForecastFlagMask) << (8u * b);
    }
    words[k] = w;
  }
  tile_sync<W>();
  // the pass reads the private slots as the object's group rows
  r3.z = base;
  r3.w = (uint32_t)C;
  const uint64_t* col = reinterpret_cast<const uint64_t*>(a.slots);
  LwsPassOut o = lws_pass_one<W, FlagLoadCoherent>(r0, r1, r2, r3, col, a.n_slots, 0u, lane);
  if (o.v1.z & (LWSE_LOUT_RUP_ERROR | LWSE_LOUT_STATUS_ERROR | LWSE_LOUT_IRREGULAR)) {
    if (!kWrite && lane == 0) a.fc[i] = lwse_lws_forecast{LWSE_LWSF_NOT_FORECAST, 0u, 0u, 0u, 0, 0, 0, 0};
    return;
  }
  const int32_t R = (int32_t)r1.x, P = (int32_t)r1.y;
  uint32_t lflags = r0.w;
  uint32_t flags = ((o.v1.z & LWSE_LOUT_COND_MASK) >> LWSE_LOUT_COND_SHIFT) == LWSE_COND_UPDATE_IN_PROGRESS
                       ? LWSE_LWSF_ROLLING
                       : 0u;
  int32_t peak = (lflags & LWSE_LWS_STS_EXISTS) ? (int32_t)r2.x : 0;
  int32_t floor_ready = (int32_t)o.v0.w;
  uint32_t n_steps = 0;
  bool stopped = false;
  // A guard, not a stop the replay reaches: after the first apply p' and n' never rise, and a cycle that
  // leaves both as they were changes nothing, so an object stops within about C cycles (DESIGN.md).
  // MAX_CYCLES binds for C >= 2^15.
  const uint32_t cap = (uint32_t)min(2 * C + 8, (long long)LWSE_LWS_FORECAST_MAX_CYCLES);
  for (uint32_t c = 0; c < cap; c++) {
    // the pass's reads of the slots (by any lane of the tile) come before this cycle's stores
    tile_sync<W>();
    const int32_t p2 = (int32_t)o.v0.x, n2 = (int32_t)o.v0.y;
    if ((long long)n2 > C) break;  // the slots cannot hold it: UNFINISHED
    peak = max(peak, n2);
    // 2. apply, and the cycle's floor before it
    uint32_t kept = 0, gained = 0;
    bool changed = false;
    for (uint32_t k = lane; k < n_words; k += W) {
      const uint64_t w = words[k];
      const int32_t off = (int32_t)(k << 3);
      const uint64_t in_n = lanes_upto((int64_t)n2 - off), ge_p = kLaneOnes & ~lanes_upto((int64_t)p2 - off);
      const uint64_t cu = (w >> 4) & kLaneOnes, cnt = (w >> 2) & kLaneOnes, crd = (w >> 3) & kLaneOnes;
      kept += __popcll(in_n & cnt & crd & ~(ge_p & ~cu));
      gained |= (uint32_t)((in_n & ~(w & crd)) != 0ull);  // STATE_READY or COND_READY missing below n'
      const uint64_t nw = in_n * 0x0Dull | ((ge_p | cu) & in_n) * 0x12ull;
      if (nw != w) {
        words[k] = nw;
        changed = true;
      }
    }
    floor_ready = min(floor_ready, tile_add<W>((int32_t)kept));
    if (c == 0 && tile_or<W>(gained)) flags |= LWSE_LWSF_WAITING;
    const uint32_t nflags = (lflags | LWSE_LWS_STS_EXISTS | LWSE_LWS_ANNOT_VALID) & ~LWSE_LWS_UPDATED;
    changed = tile_or<W>(changed ? 1u : 0u) != 0u || nflags != lflags || (int32_t)r2.x != n2 ||
              (int32_t)r2.y != p2 || (int32_t)r2.z != R;
    if (!changed) {
      stopped = true;
      break;
    }
    lflags = nflags;
    r2.x = (uint32_t)n2;
    r2.y = (uint32_t)p2;
    r2.z = (uint32_t)R;
    tile_sync<W>();
    // 1. the next pass: the state this cycle left
    o = lws_pass_one<W, FlagLoadCoherent>(make_uint4(r0.x, r0.y, r0.z, lflags), r1, r2, r3, col, a.n_slots, 0u, lane);
    if constexpr (kWrite) {
      const unsigned long long row = (unsigned long long)step_base + n_steps;
      if (lane == 0) {
        if (row < a.steps_rows)
          a.steps[row] = lwse_lws_forecast_step{(int32_t)o.v0.x, (int32_t)o.v0.y, (int32_t)o.v0.w, (int32_t)o.v1.x};
        else
          atomicAdd(a.refused, 1ull);
      }
    }
    n_steps++;
    if constexpr (kWrite) {
      if (n_steps == step_limit) return;  // every reserved row is written: the rest is the summary pass's
    }
  }
  if constexpr (!kWrite) {
    const int32_t fp = (int32_t)o.v0.x, fr = (int32_t)o.v0.y;
    if (!stopped)
      flags |= LWSE_LWSF_UNFINISHED;
    else {
      if (o.v1.z & LWSE_LOUT_UPDATE_DONE) flags |= LWSE_LWSF_DONE;
      if (fp > 0 && fp == P) flags |= LWSE_LWSF_HELD;
    }
    if (lane == 0) a.fc[i] = lwse_lws_forecast{flags, n_steps, n_steps, n_steps, peak, floor_ready, fp, fr};
  }
}

template <int W, bool kWrite>
__global__ void __launch_bounds__(256) lws_forecast_kernel(const LwsForecastArgs a) {
  constexpr uint32_t kTilesPerBlock = 256 / W;
  const uint32_t lane = threadIdx.x & (W - 1);
  const uint32_t n_tiles = gridDim.x * kTilesPerBlock;
  for (uint32_t i = blockIdx.x * kTilesPerBlock + threadIdx.x / W; i < a.n_lws; i += n_tiles)
    lws_forecast_one<W, kWrite>(a, i, lane);
}

static LwsForecastArgs forecast_args(const LwsForecastHost* h) {
  return LwsForecastArgs{h->lws,  h->n_lws, h->group_out, h->n_groups,   h->slot_off,
                         h->slots, h->n_slots, h->fc,      h->steps, h->steps_rows, h->totals + 3};
}

// The private slot layout: slot_off and totals[2].
int launch_lws_forecast_slots(const LwsForecastHost* h, int sm_count, cudaStream_t s) {
  if (h->n_lws == 0) return 0;
  const uint32_t want = (h->n_lws + 255u) / 256u, cap = (uint32_t)sm_count * 8u;
  lws_forecast_slots_kernel<<<want < cap ? want : cap, 256, 0, s>>>(forecast_args(h), h->slot_off);
  launch_forecast_scan(SlotLayoutOp{h->slot_off}, h->n_lws, h->totals + 4, h->totals + 2, nullptr, s);
  return launch_result(4);
}

template <int W, bool kWrite>
static void launch_tiles(const LwsForecastArgs& a, int sm_count, cudaStream_t s) {
  constexpr uint32_t kTilesPerBlock = 256 / W;
  const uint32_t want = (a.n_lws + kTilesPerBlock - 1) / kTilesPerBlock, cap = (uint32_t)sm_count * 8u;
  lws_forecast_kernel<W, kWrite><<<want < cap ? want : cap, 256, 0, s>>>(a);
}

template <bool kWrite>
static void launch_replay(const LwsForecastArgs& a, int sm_count, cudaStream_t s) {
  switch (pick_tile(a.n_groups, a.n_lws)) {
    case 32: launch_tiles<32, kWrite>(a, sm_count, s); break;
    case 16: launch_tiles<16, kWrite>(a, sm_count, s); break;
    case 8: launch_tiles<8, kWrite>(a, sm_count, s); break;
    case 4: launch_tiles<4, kWrite>(a, sm_count, s); break;
    case 2: launch_tiles<2, kWrite>(a, sm_count, s); break;
    default: launch_tiles<1, kWrite>(a, sm_count, s); break;
  }
}

// write_pass = false: the summary pass and the scan.  write_pass = true: the write pass into h->steps,
// which holds the rows the scan counted as written.  Both on stream s.
int launch_lws_forecast(const LwsForecastHost* h, bool write_pass, int sm_count, cudaStream_t s) {
  if (h->n_lws == 0) return 0;
  const LwsForecastArgs a = forecast_args(h);
  int launched;
  if (write_pass) {
    launch_replay<true>(a, sm_count, s);
    launched = 1;
  } else {
    launch_replay<false>(a, sm_count, s);
    launch_forecast_scan(StepLayoutOp<lwse_lws_forecast, LWSE_LWSF_TRUNCATED>{h->fc, h->step_capacity, h->want_steps ? 1 : 0},
                         h->n_lws, h->totals + 4, h->totals + 0, h->totals + 1, s);
    launched = 4;
  }
  return launch_result(launched);
}

}  // namespace lwse
