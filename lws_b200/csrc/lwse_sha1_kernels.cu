// SHA-1 group / subgroup keys (sm_90a): one lane per key string, a warp per 32 consecutive keys.
//
// pkg/webhooks/pod_webhook.go:180-182 genGroupUniqueKey = Sha1Hash("<ns>/<podName>")
// and :130,:151 Sha1Hash("<leaderName>/<subGroupIndex>"); pkg/utils/utils.go:39-43
// Sha1Hash = hex(crypto/sha1).  The engine emits the 20 raw digest bytes; the
// caller hex-encodes (the label value is the 40-character hex string).
// FIPS 180-4 SHA-1, big-endian message schedule kept in a 16-word ring.
//
// Memory side: the 32 strings of a warp are one contiguous byte range of the blob (string i
// starts where i-1 ends), so the warp copies that range into shared memory with coalesced
// 32-bit loads and every lane assembles its message words from there; the 20-byte digests leave
// through shared memory too, as 160 consecutive words per warp.  (Per-thread byte loads touched
// eight sectors per load instruction and wrote 20 single bytes per key.)
// The subgroup form appends "/<index>" itself: getSubGroupIndex (:249-255) is evaluated on the
// device, in C's truncating division like Go's, and the decimal suffix never exists in memory.
#include "lwse_device.cuh"
#include "lwse_launch.cuh"

namespace lwse {

__device__ __forceinline__ uint32_t rotl(uint32_t x, int n) { return __funnelshift_l(x, x, n); }

__device__ __forceinline__ void sha1_block(uint32_t* h, uint32_t* w) {
  uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4];
#pragma unroll
  for (int t = 0; t < 80; t++) {
    if (t >= 16) {
      const uint32_t x = w[(t - 3) & 15] ^ w[(t - 8) & 15] ^ w[(t - 14) & 15] ^ w[t & 15];
      w[t & 15] = rotl(x, 1);
    }
    uint32_t f, k;
    if (t < 20) {
      f = (b & c) | (~b & d);
      k = 0x5A827999u;
    } else if (t < 40) {
      f = b ^ c ^ d;
      k = 0x6ED9EBA1u;
    } else if (t < 60) {
      f = (b & c) | (b & d) | (c & d);
      k = 0x8F1BBCDCu;
    } else {
      f = b ^ c ^ d;
      k = 0xCA62C1D6u;
    }
    const uint32_t tmp = rotl(a, 5) + f + e + k + w[t & 15];
    e = d;
    d = c;
    c = rotl(b, 30);
    b = a;
    a = tmp;
  }
  h[0] += a;
  h[1] += b;
  h[2] += c;
  h[3] += d;
  h[4] += e;
}

constexpr uint32_t kShaWarps = 4;          // warps per CTA
constexpr uint32_t kShaStageBytes = 3072;  // staged blob bytes per warp (32 keys of up to 96 bytes on average)

struct Sha1Args {
  const uint8_t* bytes;
  const uint32_t* offsets;
  uint32_t n;
  uint8_t* digests;
  // subgroup form (all null / 0 for plain keys)
  const int32_t* pod_count;
  const int32_t* subgroup_size;
  const int32_t* worker_index;
  int32_t* index_out;
};

// pod_webhook.go:249-255 getSubGroupIndex, Go's truncating `/` and `%`
__device__ __forceinline__ int32_t sub_group_index(int32_t pod_count, int32_t sg, int32_t worker_index) {
  if ((pod_count - 1) % sg == 0) return (worker_index - 1) / sg;
  return worker_index / sg;
}

template <bool kSubgroup>
__global__ void __launch_bounds__(kShaWarps * 32) sha1_kernel(const Sha1Args a) {
  __shared__ uint32_t s_stage[kShaWarps][kShaStageBytes / 4 + 2];
  __shared__ uint32_t s_out[kShaWarps][160];
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint32_t n_warps = gridDim.x * kShaWarps;
  for (uint32_t k0 = (blockIdx.x * kShaWarps + warp) * 32u; k0 < a.n; k0 += n_warps * 32u) {
    const uint32_t i = k0 + lane;
    const bool live = i < a.n;
    const uint32_t begin = live ? __ldg(a.offsets + i) : 0u, end = live ? __ldg(a.offsets + i + 1) : 0u;
    // the warp's contiguous byte range, staged with aligned 32-bit loads
    const uint32_t last_key = min(k0 + 31u, a.n - 1u);
    const uint32_t r0 = __shfl_sync(0xFFFFFFFFu, begin, 0);
    const uint32_t r1 = __shfl_sync(0xFFFFFFFFu, end, (int)(last_key - k0));
    const uint32_t w0 = r0 >> 2, w1 = (r1 + 3u) >> 2;  // 32-bit words of the blob
    const bool staged = (w1 - w0) * 4u <= kShaStageBytes && ((reinterpret_cast<uintptr_t>(a.bytes) & 3u) == 0);
    if (staged) {
      const uint32_t* src = reinterpret_cast<const uint32_t*>(a.bytes);
      for (uint32_t w = w0 + lane; w < w1; w += 32u) s_stage[warp][w - w0] = __ldg(src + w);
    }
    __syncwarp();
    const uint8_t* sb = reinterpret_cast<const uint8_t*>(s_stage[warp]) - (size_t)w0 * 4u;  // sb[p] = blob byte p
    auto byte_at = [&](uint32_t p) -> uint32_t { return staged ? sb[p] : __ldg(a.bytes + p); };

    // the message: string bytes, then (subgroup form) "/" and the decimal index
    uint8_t suffix[12];
    uint32_t n_suffix = 0;
    int32_t index = 0;
    bool bad = false;
    if (kSubgroup && live) {
      const int32_t sg = __ldg(a.subgroup_size + i);
      if (sg == 0) {
        bad = true;  // Go panics on the division; the row is flagged
        index = INT32_MIN;
      } else {
        index = sub_group_index(__ldg(a.pod_count + i), sg, __ldg(a.worker_index + i));
        suffix[n_suffix++] = '/';
        uint32_t mag = index < 0 ? (uint32_t)(-(int64_t)index) : (uint32_t)index;
        if (index < 0) suffix[n_suffix++] = '-';
        uint8_t dig[10];
        int nd = 0;
        do {
          dig[nd++] = (uint8_t)('0' + mag % 10u);
          mag /= 10u;
        } while (mag);
        while (nd) suffix[n_suffix++] = dig[--nd];
      }
      a.index_out[i] = index;
    }
    const uint32_t slen = end - begin, len = slen + n_suffix;
    uint32_t h[5] = {0x67452301u, 0xEFCDAB89u, 0x98BADCFEu, 0x10325476u, 0xC3D2E1F0u};
    if (live && !bad) {
      uint32_t w[16];
      // message bytes, then 0x80, zeros, and the 64-bit big-endian bit length
      const uint32_t total = ((len + 8u) / 64u + 1u) * 64u;
      for (uint32_t pos = 0; pos < total; pos += 64u) {
#pragma unroll
        for (int j = 0; j < 16; j++) {
          uint32_t word = 0;
#pragma unroll
          for (int b = 0; b < 4; b++) {
            const uint32_t p = pos + (uint32_t)j * 4u + (uint32_t)b;
            uint32_t byte;
            if (p < slen)
              byte = byte_at(begin + p);
            else if (p < len)
              byte = suffix[p - slen];
            else if (p == len)
              byte = 0x80u;
            else
              byte = 0u;
            word = (word << 8) | byte;
          }
          w[j] = word;
        }
        if (pos + 64u == total) {
          w[14] = len >> 29;  // bit length, high word
          w[15] = len << 3;
        }
        sha1_block(h, w);
      }
    } else {
#pragma unroll
      for (int j = 0; j < 5; j++) h[j] = 0u;
    }
    // digests: 5 big-endian words per key, written as 160 consecutive words per warp
    __syncwarp();
#pragma unroll
    for (int j = 0; j < 5; j++) s_out[warp][lane * 5u + (uint32_t)j] = __byte_perm(h[j], 0u, 0x0123);
    __syncwarp();
    const uint32_t keys_here = min(32u, a.n - k0);
    if ((reinterpret_cast<uintptr_t>(a.digests) & 3u) == 0) {
      uint32_t* dst = reinterpret_cast<uint32_t*>(a.digests) + (size_t)k0 * 5u;
      for (uint32_t q = lane; q < keys_here * 5u; q += 32u) dst[q] = s_out[warp][q];
    } else if (live) {
      const uint8_t* src = reinterpret_cast<const uint8_t*>(&s_out[warp][lane * 5u]);
      for (uint32_t q = 0; q < 20u; q++) a.digests[(size_t)i * 20u + q] = src[q];
    }
    __syncwarp();
  }
}

static int launch_sha1_form(const Sha1Args& a, bool subgroup, int sm_count, cudaStream_t s) {
  if (a.n == 0) return 0;
  const uint32_t want = (a.n + kShaWarps * 32u - 1u) / (kShaWarps * 32u);
  const uint32_t cap = (uint32_t)sm_count * 16u;
  const unsigned grid = want < cap ? want : cap;
  if (subgroup)
    sha1_kernel<true><<<grid, kShaWarps * 32, 0, s>>>(a);
  else
    sha1_kernel<false><<<grid, kShaWarps * 32, 0, s>>>(a);
  return launch_result(1);
}

int launch_sha1(const uint8_t* d_bytes, const uint32_t* d_offsets, uint32_t n, uint8_t* d_digests,
                int sm_count, cudaStream_t s) {
  Sha1Args a{d_bytes, d_offsets, n, d_digests, nullptr, nullptr, nullptr, nullptr};
  return launch_sha1_form(a, false, sm_count, s);
}

int launch_subgroup_keys(const uint8_t* d_bytes, const uint32_t* d_offsets, uint32_t n, const int32_t* d_pod_count,
                         const int32_t* d_subgroup_size, const int32_t* d_worker_index, int32_t* d_index_out,
                         uint8_t* d_digests, int sm_count, cudaStream_t s) {
  Sha1Args a{d_bytes, d_offsets, n, d_digests, d_pod_count, d_subgroup_size, d_worker_index, d_index_out};
  return launch_sha1_form(a, true, sm_count, s);
}

}  // namespace lwse
