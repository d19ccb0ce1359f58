// Peer exchange for the multi-GPU placement step (sm_90a, NVLink / NVSwitch peer memory).
//
// A placement step needs every shard's [per-node occupancy | request rows].  Instead of a NCCL
// all-gather (launch + protocol latency of the order of the sweep itself for a few tens of KB),
// every rank PUSHES its part straight into every peer's gathered buffer with peer stores over
// NVLink and then raises a per-source flag there; the same kernel's last CTA then waits until the
// flags of all sources have reached this step.  One launch per rank and step, no host round trip,
// no collective library on the data path.
//
// Buffers (one cudaMalloc per rank, exported with cudaIpcGetMemHandle, opened by every peer):
//   [buffer 0: world x part_stride][buffer 1][buffer 2][flags: world x 8 B][ticket][error]
// Step s uses buffer s % 3.  Two ways to wait:
//   - in step   (wait_step = s): the round of step s reads the parts every rank pushed for step s;
//   - lagged    (wait_step = s - 1): the round of step s reads buffer (s - 1) % 3, the parts of the
//     PREVIOUS step (own part included: every rank sees the same snapshot).  Nobody waits for the
//     slowest rank's launch of this step — the flags of s - 1 were raised a whole tick ago — so the
//     ranks stay only loosely coupled (one tick of slack absorbs launch skew).
// Three buffers make both safe: rank A writes buffer s % 3 only after every rank raised its flag
// for s - 1 (A's own wait of tick s - 1 or s), i.e. after every rank B has enqueued push(s - 1),
// which on B's stream comes after B's round of tick s - 2 — the last reader of buffer (s - 3) % 3
// = s % 3.
#include "lwse_device.cuh"
#include "lwse_launch.cuh"

namespace lwse {

struct ExchangeArgs {
  const uint4* local_part;         // this rank's part (16-byte aligned), part_bytes
  uint8_t* const* peer_base;       // device array: base of every rank's exchange buffer (own included)
  unsigned long long* flags;       // local: flags[src] = last step src has pushed here
  uint32_t* ticket;                // local: CTA completion counter
  uint32_t* error;                 // local: set to 1 when the wait timed out
  uint64_t part_bytes, part_stride, half_bytes, flags_offset;
  uint64_t step, wait_step;        // step == 0: this launch is a node of a replayed graph — the step is the
                                   // device counter + 1 (the host counts the same calls), lagged as below
  unsigned long long* step_ctr;    // local: the step of the last push (every launch stores its step there)
  uint32_t lagged;
  uint32_t world, rank;
  uint64_t timeout_ns;
};

__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

__global__ void __launch_bounds__(256) exchange_push_kernel(const ExchangeArgs a) {
  __shared__ uint32_t s_last;
  pdl_launch_dependents();  // the placement round may take its SMs now; it waits for this grid to complete
  uint64_t step = a.step, wait_step = a.wait_step;
  if (step == 0ull) {  // (every CTA reads the counter before the last one — the last to finish — advances it)
    step = *reinterpret_cast<volatile unsigned long long*>(a.step_ctr) + 1ull;
    wait_step = (a.lagged && step > 1ull) ? step - 1ull : step;
  }
  const uint64_t n_vec = a.part_bytes >> 4;
  const uint64_t dst_off = (step % 3ull) * a.half_bytes + (uint64_t)a.rank * a.part_stride;
  // every peer's copy of this rank's part: the loads of the local part are shared by all targets
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint4 v = __ldg(a.local_part + i);
    for (uint32_t p = 0; p < a.world; p++) reinterpret_cast<uint4*>(a.peer_base[p] + dst_off)[i] = v;
  }
  __threadfence_system();  // this thread's peer stores are visible system-wide before the ticket
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(a.ticket, 1u) == gridDim.x - 1u ? 1u : 0u;
  __syncthreads();
  if (!s_last) return;
  // last CTA: every CTA's stores are out (each fenced before taking its ticket)
  __threadfence_system();
  if (threadIdx.x == 0) {
    *a.ticket = 0u;  // ready for the next launch (stream-ordered)
    *a.step_ctr = step;
  }
  if (threadIdx.x < a.world) {
    unsigned long long* peer_flags = reinterpret_cast<unsigned long long*>(a.peer_base[threadIdx.x] + a.flags_offset);
    st_release_sys(peer_flags + a.rank, step);
    // … and wait for source threadIdx.x to have pushed this step here
    unsigned long long t0;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    while (ld_acquire_sys(a.flags + threadIdx.x) < wait_step) {
      unsigned long long t;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      if (t - t0 > a.timeout_ns) {  // a peer is gone: do not hang the GPU, report
        *a.error = 1u;
        break;
      }
    }
  }
}

int launch_exchange_push(const void* d_local_part, uint8_t* const* d_peer_base, void* d_local_base,
                         uint64_t part_bytes, uint64_t part_stride, uint64_t half_bytes, uint64_t flags_offset,
                         uint64_t step, uint64_t wait_step, uint32_t world, uint32_t rank, cudaStream_t s,
                         bool lagged) {
  ExchangeArgs a{};
  uint8_t* base = static_cast<uint8_t*>(d_local_base);
  a.local_part = static_cast<const uint4*>(d_local_part);
  a.peer_base = d_peer_base;
  a.flags = reinterpret_cast<unsigned long long*>(base + flags_offset);
  a.ticket = reinterpret_cast<uint32_t*>(base + flags_offset + (uint64_t)world * 8u);
  a.error = a.ticket + 1;
  a.step_ctr = reinterpret_cast<unsigned long long*>(base + flags_offset + (uint64_t)world * 8u + 16u);
  a.lagged = lagged ? 1u : 0u;
  a.part_bytes = part_bytes;
  a.part_stride = part_stride;
  a.half_bytes = half_bytes;
  a.flags_offset = flags_offset;
  a.step = step;
  a.wait_step = wait_step;
  a.world = world;
  a.rank = rank;
  a.timeout_ns = 2000000000ull;
  const uint64_t n_vec = part_bytes >> 4;
  unsigned grid = (unsigned)((n_vec + 255) / 256);
  if (grid > 32u) grid = 32u;
  if (grid < 1u) grid = 1u;
  exchange_push_kernel<<<grid, 256, 0, s>>>(a);
  return launch_result(1);
}

}  // namespace lwse
