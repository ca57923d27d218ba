// Philox4x32-10 (Salmon et al., SC'11) and the dropout keep-bit rule shared with oracle/philox.py:
//   keep(seed, frame, layer, n, pix, c) = bit (c & 31) of word ((c >> 5) & 3) of
//     philox(ctr = (pix, n | layer << 16 | (c >> 7) << 24, frame_lo, frame_hi), key = (seed_lo, seed_hi))
// Stands in for the reference's unseeded Bernoulli stream (caffe dropout_layer.cpp:37-42 / .cu:9-35).
#pragma once
#include <cstdint>

namespace sivo {

__host__ __device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                                       uint32_t k0, uint32_t k1, uint32_t out[4]) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint64_t p0 = 0xD2511F53ull * c0;
    uint64_t p1 = 0xCD9E8D57ull * c2;
    uint32_t n0 = static_cast<uint32_t>(p1 >> 32) ^ c1 ^ k0;
    uint32_t n2 = static_cast<uint32_t>(p0 >> 32) ^ c3 ^ k1;
    c1 = static_cast<uint32_t>(p1);
    c3 = static_cast<uint32_t>(p0);
    c0 = n0;
    c2 = n2;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

// The same with the sample / layer part of the counter word given whole: nl = n | layer << 16 (n < 2^16, so a caller may add
// a sample offset to it).  The fields are disjoint, so the group is added rather than or-ed: the same word, and in the
// convolution epilogue one IADD3 with the caller's addition (no extra register pressure).
__host__ __device__ __forceinline__ void dropout_bits128_nl(uint64_t seed, uint64_t frame, uint32_t nl, uint32_t pix, int g,
                                                            uint32_t out[4]) {
  philox4x32_10(pix, nl + (static_cast<uint32_t>(g) << 24), static_cast<uint32_t>(frame), static_cast<uint32_t>(frame >> 32),
                static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32), out);
}

// 128 keep bits for channels [128*g, 128*g+128) of pixel `pix` in sample `n` of dropout layer `layer`
__host__ __device__ __forceinline__ void dropout_bits128(uint64_t seed, uint64_t frame, int layer, int n,
                                                         uint32_t pix, int g, uint32_t out[4]) {
  dropout_bits128_nl(seed, frame, static_cast<uint32_t>(n) | (static_cast<uint32_t>(layer) << 16), pix, g, out);
}

}  // namespace sivo
