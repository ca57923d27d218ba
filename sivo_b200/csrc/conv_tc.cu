// Hopper (sm_90a) implicit-GEMM convolution on wgmma -- replaces cuDNN's fp32 `cudnnConvolutionForward`
// (caffe/src/caffe/layers/cudnn_conv_layer.cu:21-37) and the layers fused around it for every SegNet convolution
// (Basic: all eight 7x7 layers + the 1x1 classifier; Standard: all 26 3x3 layers).
//
// GEMM view per CTA:  D[128 pixels x N couts] += A[128 pixels x 64 cin] * B[64 cin x N couts]  per filter tap,
// M = 128 consecutive pixels of one output row, two output rows -- a "row block" -- per accumulator set.
//
//  * Activations are NHWC half, so one pixel's 64 input channels are one 128-byte row: exactly a SWIZZLE_128B K-major
//    wgmma operand row.  A TMA box {64 ch, 128+K-1 px, 1 row} of the input lands one *halo row* in shared memory;
//    out-of-image coordinates are zero-filled by TMA = the conv's zero padding.
//  * The A operand of tap (kh, kw) for output row r is the same halo row shifted by kw pixels: the shared-memory matrix
//    descriptor simply starts kw*128 bytes later (the swizzle phase follows the absolute address), so each input row is
//    fetched from L2 once per K rows of output instead of K*K times.
//  * A CTA walks down a 128-px-wide column strip one row block at a time with a ring of halo rows (mbarrier full / empty
//    pairs): every input row is loaded once per CTA (plus the K-1 overlap between vertically adjacent CTAs) and released
//    as soon as its last tap row has retired.
//  * Weights stream through a TMA ring, one {64 cin x N cout} tile per tap, [tap][cout][cin].
//  * The 3-channel first layer reads a window-folded view of the zero-padded 8-channel image (KW = 1, see conv_tc_plan).
//  * 384 threads = three warpgroups.  Warpgroup 0 produces (warp 0: halo rows, warp 1: weights; setmaxnreg 40);
//    warpgroups 1 and 2 consume (setmaxnreg 232): consumer g owns pixels [64 g, 64 g + 64) of the tile, issues the
//    m64nNk16 wgmma of both rows of the block into register accumulators, and runs the epilogue on them -- bias / BN
//    affine / ReLU -> half, then store | dropout | max-unpool scatter | 2x2 max-pool + argmax | 1x1 classifier -> float
//    logits -- while the other consumer's MMAs keep the tensor core busy.
//  * Constants (bias, BN, classifier weights) are kernel parameters: the epilogue reads them from the constant bank and
//    leaves the shared-memory data path to the MMA operand reads.
#include <cuda.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <vector>

#include "philox.cuh"
#include "segnet.h"

namespace sivo {

namespace {

constexpr int kTcThreads = 3 * 128;  // warpgroup 0: TMA producers, warpgroups 1-2: wgmma consumers + epilogue
constexpr int kRows = 2;             // output rows per row block (accumulator set)
constexpr int kSlotBytes = 17 * 1024;  // one halo row: (128 + K - 1) px * 128 B, padded to a 1024-B multiple
constexpr int kMaxBStages = 6;
constexpr int kEmptyArrivals = 8;    // every consumer warp releases a ring slot once its MMAs that read it retired

struct TcParams {
  int H, W, N_batch;       // spatial size and batch of input == output
  int cout_total;          // channel stride of the output tensor
  int n_tile;              // wgmma N (16 for the float logits layer, else 64 or 128)
  int chunks;              // Cin / 64
  int b_stages;            // weight ring depth (as many of kMaxBStages as fit in shared memory)
  int out_f32;             // 1: 16-channel float output (logits); 2: n_tile-wide float output (split-operand fp32 mode)
  int split;               // split-operand fp32 mode: A = [hi Cin | lo Cin] half planes of the float input, B K-axis = per real chunk
                           // [W_hi | W_lo | W_hi]; `chunks` then counts A chunks (2 * Cin / 64: hi and lo of each, interleaved)
  int cin_real;            // Cin (split mode: channel offset of the lo plane)
  float acc_scale;         // split mode: the weights were scaled by a power of two before the hi/lo split; 1 / that
  float rz_comp;           // split mode: expected truncation loss per accumulate step relative to the running sum (see seg_rows);
                           // each flushed segment of m steps is scaled by 1 + rz_comp * m before it is added (0 = off)
  int seg_rows;            // split mode: tap rows per accumulation segment.  The tensor core adds into its fp32 accumulator with
                           // truncation towards zero, so the loss grows linearly with the chain length; the block's MMAs are
                           // therefore cut into segments of (A chunk, seg_rows tap rows) that each start a fresh accumulator,
                           // and the epilogue sums the segments in registers with round-to-nearest adds.
  int pairs_per_cta;       // row blocks one CTA walks
  int strips;              // ceil(W / 128)
  int relu, has_bn, has_drop;
  float slope;
  void* out;
  // dropout fused into the epilogue (decoder convs of Basic: decdrop4 / decdrop3)
  uint64_t seed;
  const uint64_t* frame;
  int drop_layer;
  float drop_scale;
  // max-unpool fused into the epilogue (decoder convs): the output tensor is 2H x 2W and every pixel's channel
  // lands in the 2x2 position its pooling mask names, zeros elsewhere (upsample_layer.cpp:74-103)
  const uint8_t* unpool_mask;
  int mask_n;
  // 2x2/2 max pool with argmax fused into the epilogue (encoder convs): only the pooled tensor and its 2-bit mask are
  // written (pooling_layer.cpp:140-187: scan (0,0),(0,1),(1,0),(1,1), strict '>', so the first maximum wins)
  __half* pool_out;        // [N][H/2][W/2][cout_total]
  uint8_t* pool_mask;      // same shape
  // 1x1 classifier fused into the epilogue (the layer feeding Softmax): logits[j] = cls_b[j] + sum_c half(out[c]) * cls_w[c][j];
  // the 64-channel output itself is then never written
  int has_cls;
  float* cls_out;          // [N][H][W][16]
};

// Per-layer constants, passed by value as a kernel parameter so that the epilogue reads them from the constant bank.
constexpr int kMaxCout = 512;
struct TcConsts {
  float bias[kMaxCout], bn_scale[kMaxCout], bn_shift[kMaxCout];
  float cls_w[64 * 16];    // fused classifier: [cin][16] float (half-rounded values), j >= classes zero
  float cls_b[16];
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Bounded wait: a protocol bug must surface as a CUDA error, never as a hung GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t addr = smem_u32(bar);
  for (uint32_t spin = 0;; ++spin) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
    if (done) return;
    if (spin > (1u << 26)) asm volatile("trap;");
  }
}

__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// K-major SWIZZLE_128B wgmma matrix descriptor: rows of 128 B, 8-row groups 1024 B apart.  High word: stride byte offset
// 1024 >> 4 (bits 32-45), base offset 0 (bits 49-51), layout SWIZZLE_128B = 1 (bits 62-63).  Low word: start address >> 4
// (bits 0-13), leading byte offset 1 (unused by swizzled K-major layouts).  A K step of 16 halfs advances the start by
// 32 B (>> 4: 2); a tap column shifts an A operand by one 128-B row (8).  The XOR phase of the swizzle follows the
// absolute shared-memory address, as TMA wrote it, so an operand may start at any 128-B row of a 1024-B-aligned halo row.
constexpr uint32_t kDescHi = (1024u >> 4) | (1u << 30);
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr) {
  return (static_cast<uint64_t>(kDescHi) << 32) | (((smem_addr & 0x3FFFFu) >> 4) | (1u << 16));
}

// D[64 x N] (+)= A[64 x 16] * B[16 x N], both operands K-major in shared memory, fp32 accumulators in registers
// (fragment layout: d[4 j + 2 h + e] = row 16 warp + lane / 4 + 8 h, column 8 j + 2 (lane % 4) + e)
__device__ __forceinline__ void wgmma(float (&d)[8], uint64_t a, uint64_t b) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, 1, 1, 1, 0, 0;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(a), "l"(b));
}
__device__ __forceinline__ void wgmma(float (&d)[32], uint64_t a, uint64_t b) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, 1, 1, 1, 0, 0;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b));
}
__device__ __forceinline__ void wgmma(float (&d)[64], uint64_t a, uint64_t b) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, "
      "%47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, 1, 1, 1, 0, 0;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
        "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
        "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
        "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
        "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Ties the accumulator registers to the preceding wait: the compiler must not move their reads (or the zeroing of a
// fresh segment) across it.
template <int R, int F>
__device__ __forceinline__ void fence_acc(float (&d)[R][F]) {
#pragma unroll
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int i = 0; i < F; ++i) asm volatile("" : "+f"(d[r][i])::"memory");
}

__device__ __forceinline__ float affine(const TcParams& p, const TcConsts& cst, float v, int c) {
  float t = __fadd_rn(v, cst.bias[c]);
  if (p.has_bn) t = __fadd_rn(__fmul_rn(t, cst.bn_scale[c]), cst.bn_shift[c]);
  if (p.relu) t = t > 0.f ? t : __fmul_rn(p.slope, t);
  return t;
}

// Fused 1x1 classifier, one quad lane's share: partial logits over its 16 channels (8 j + 2 Q + e) of pixel h.
template <int Q>
__device__ __forceinline__ void cls_partial(const TcParams& p, const TcConsts& cst, const float (&a)[32], int h, float (&l)[16]) {
#pragma unroll
  for (int jj = 0; jj < 16; ++jj) l[jj] = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int c = 8 * j + 2 * Q + e;
      const float hv = __half2float(__float2half_rn(affine(p, cst, a[4 * j + 2 * h + e], c)));
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) l[jj] = fmaf(hv, cst.cls_w[c * 16 + jj], l[jj]);
    }
}

// Epilogue of one row block for one consumer thread.  The thread holds, per output row r, pixels m0 and m0 + 8 of its
// consumer's 64 (h = 0, 1) and channels 8 j + 2 q + e (q = lane % 4) of each: acc[r][4 j + 2 h + e].  `x_m0` = image column
// of pixel m0, `y0` = first row of the block, `n0` = first output channel of the CTA's tile.  Called by all 32 lanes
// (warp shuffles); out-of-image pixels are masked at the stores.
template <int N>
__device__ __forceinline__ void epilogue_block(const TcParams& p, const TcConsts& cst, const float (&acc)[kRows][N / 2], int img,
                                               int y0, int x_m0, int n0, int lane) {
  const int q = lane & 3;
  const bool img_ok = img < p.N_batch;  // img >= N: the odd image out of an image-pair tile (PK2)
  if (p.pool_out) {  // both rows of the block: 2x2 max with first-maximum argmax; the horizontal neighbour is pixel m + 1 = lane ^ 4
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int x = x_m0 + 8 * h;
      const bool writer = ((x & 1) == 0) && y0 + 1 < p.H && x + 1 < p.W && img_ok;
      const size_t o = ((static_cast<size_t>(img) * (p.H >> 1) + (y0 >> 1)) * (p.W >> 1) + (x >> 1)) * p.cout_total + n0;
#pragma unroll
      for (int j = 0; j < N / 8; ++j) {
        const int c = 8 * j + 2 * q;
        const __half2 ha = __floats2half2_rn(affine(p, cst, acc[0][4 * j + 2 * h], n0 + c), affine(p, cst, acc[0][4 * j + 2 * h + 1], n0 + c + 1));
        const __half2 hc = __floats2half2_rn(affine(p, cst, acc[1][4 * j + 2 * h], n0 + c), affine(p, cst, acc[1][4 * j + 2 * h + 1], n0 + c + 1));
        const uint32_t a = *reinterpret_cast<const uint32_t*>(&ha), cc = *reinterpret_cast<const uint32_t*>(&hc);
        const uint32_t b = __shfl_xor_sync(0xffffffffu, a, 4), d = __shfl_xor_sync(0xffffffffu, cc, 4);
        // window in scan order: a = (y, x), b = (y, x+1), c = (y+1, x), d = (y+1, x+1); two channels per register
        uint32_t best = a, arg = 0;
        const uint32_t cand[3] = {b, cc, d};
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          // strict '>' per half (false on NaN, like __hgt): 0xFFFF where the candidate wins
          const uint32_t sel = __hgt2_mask(*reinterpret_cast<const __half2*>(&cand[k]), *reinterpret_cast<const __half2*>(&best));
          best = (best & ~sel) | (cand[k] & sel);
          const uint32_t selb = __byte_perm(sel, 0u, 0x4420);  // the two half masks as two byte masks (bytes 0 and 1)
          arg = (arg & ~selb) | ((0x0101u * static_cast<uint32_t>(k + 1)) & selb);
        }
        if (writer) {
          *reinterpret_cast<uint32_t*>(p.pool_out + o + c) = best;
          *reinterpret_cast<uint16_t*>(p.pool_mask + o + c) = static_cast<uint16_t>(arg);
        }
      }
    }
    return;
  }
#pragma unroll
  for (int r = 0; r < kRows; ++r) {
    const int y = y0 + r;
    const bool row_ok = y < p.H && img_ok;
    if constexpr (N == 64) if (p.has_cls) {  // conv (+bias) -> half rounding (as the unfused path stores it) -> 1x1 classifier -> float logits
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float l[16];
        switch (q) {  // one copy per quad lane, so that the classifier weights are compile-time constant-bank operands
          case 0: cls_partial<0>(p, cst, acc[r], h, l); break;
          case 1: cls_partial<1>(p, cst, acc[r], h, l); break;
          case 2: cls_partial<2>(p, cst, acc[r], h, l); break;
          default: cls_partial<3>(p, cst, acc[r], h, l); break;
        }
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {  // the four lanes of a pixel hold a quarter of its channels each
          l[jj] += __shfl_xor_sync(0xffffffffu, l[jj], 1);
          l[jj] += __shfl_xor_sync(0xffffffffu, l[jj], 2);
          l[jj] = __fadd_rn(l[jj], cst.cls_b[jj]);
        }
        const int x = x_m0 + 8 * h;
        const float4 v = q == 0 ? make_float4(l[0], l[1], l[2], l[3]) : q == 1 ? make_float4(l[4], l[5], l[6], l[7])
                       : q == 2 ? make_float4(l[8], l[9], l[10], l[11]) : make_float4(l[12], l[13], l[14], l[15]);
        if (row_ok && x < p.W) *reinterpret_cast<float4*>(p.cls_out + ((static_cast<size_t>(img) * p.H + y) * p.W + x) * 16 + 4 * q) = v;
      }
      continue;
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int x = x_m0 + 8 * h;
      const bool inside = row_ok && x < p.W;
      const size_t pix = (static_cast<size_t>(img) * p.H + y) * p.W + x;
      if (p.out_f32) {  // float logits / split-mode output (the split epilogue passes accumulators already scaled by 2^-s)
#pragma unroll
        for (int j = 0; j < N / 8; ++j) {
          const int c = n0 + 8 * j + 2 * q;
          const float2 v = make_float2(affine(p, cst, acc[r][4 * j + 2 * h], c), affine(p, cst, acc[r][4 * j + 2 * h + 1], c + 1));
          if (inside) *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.out) + pix * p.cout_total + c) = v;
        }
        continue;
      }
      uint32_t bits[4] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu};
      if (p.has_drop && inside)  // a tile never straddles a 128-channel group (n0 is a multiple of N <= 128)
        dropout_bits128(p.seed, *p.frame, p.drop_layer, img, static_cast<uint32_t>(y * p.W + x), n0 >> 7, bits);
      const size_t mask_pix = (static_cast<size_t>(img % p.mask_n) * p.H + y) * p.W + x;
#pragma unroll
      for (int j = 0; j < N / 8; ++j) {
        const int c = n0 + 8 * j + 2 * q;
        __half2 hv = __floats2half2_rn(affine(p, cst, acc[r][4 * j + 2 * h], c), affine(p, cst, acc[r][4 * j + 2 * h + 1], c + 1));
        if (p.has_drop) {  // y = x * keep * 2 on the stored half value (exact)
          const int wsel = (c >> 5) & 3;  // selects, not a dynamically indexed (= local-memory) array
          const uint32_t keep = wsel == 0 ? bits[0] : wsel == 1 ? bits[1] : wsel == 2 ? bits[2] : bits[3];
          const int bit = c & 31;
          hv = __hmul2(hv, __floats2half2_rn((keep >> bit) & 1u ? p.drop_scale : 0.f, (keep >> (bit + 1)) & 1u ? p.drop_scale : 0.f));
        }
        const uint32_t w = *reinterpret_cast<const uint32_t*>(&hv);
        if (!inside) continue;
        if (p.unpool_mask) {
          // the value goes to the 2x2 position its mask byte names, zeros to the other three
          const uint32_t m = __ldg(reinterpret_cast<const uint16_t*>(p.unpool_mask + mask_pix * p.cout_total + c));
          __half* const ob = static_cast<__half*>(p.out) + ((static_cast<size_t>(img) * 2 * p.H + 2 * y) * (2 * p.W) + 2 * x) * p.cout_total + c;
          const size_t row_step = static_cast<size_t>(2 * p.W) * p.cout_total;
#pragma unroll
          for (int pos = 0; pos < 4; ++pos) {
            const uint32_t sel = ((m & 0xFFu) == static_cast<uint32_t>(pos) ? 0x0000FFFFu : 0u) | ((m >> 8) == static_cast<uint32_t>(pos) ? 0xFFFF0000u : 0u);
            *reinterpret_cast<uint32_t*>(ob + (pos >> 1) * row_step + (pos & 1) * p.cout_total) = w & sel;
          }
        } else {
          *reinterpret_cast<uint32_t*>(static_cast<__half*>(p.out) + pix * p.cout_total + c) = w;
        }
      }
    }
  }
}

// ROLL = true : one 64-channel chunk (Cin == 64); halo rows persist in the ring while the CTA walks down its
//               strip, so each input row is fetched once per CTA.
// ROLL = false: Cin = 64 * NC; per (row block, chunk) the kRows+K-1 halo rows of that chunk are fetched, used by
//               the K*K taps and released; the ring double-buffers chunks.
// KW < K : the kernel is K x KW over a *window-folded* input (KW = 1: every pixel's 64 "channels" are the 8-pixel x
//               8-channel window starting at it, so a 3-channel K x K layer is a K x 1 layer; see conv_tc_plan).
// PK2 (only with !ROLL): layers at most 64 pixels wide (Standard's conv5_x at 22x64) would fill half of every 128-pixel M tile.
//               Two images share a tile instead (consumer 0: image 2z, consumer 1: image 2z+1), and because the kw shift of a
//               shared-memory row would run from one image into the other, the shift is done by TMA: per (chunk, kw) the halo rows
//               are fetched as two 64-pixel boxes starting at pixel kw - 1 (out-of-range pixels and images zero-filled), so the
//               A operand of tap (kh, kw) is an unshifted, fully populated tile.  3x the halo traffic, which these small layers
//               have to spare; weights arrive in (kw, kh) order.
// SPLIT: split-operand fp32 mode (see TcParams::split / seg_rows); N <= 64 so that the segment sums fit in registers.
template <int K, bool ROLL, int KW, bool PK2, int N, bool SPLIT>
__global__ void __launch_bounds__(kTcThreads, 1)
k_conv_tc(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const __grid_constant__ TcParams p,
          const __grid_constant__ TcConsts cst) {
  asm volatile("griddepcontrol.launch_dependents;");  // the next kernel's CTAs may be scheduled as soon as all of ours have started
  static_assert(!PK2 || (!ROLL && KW == K), "image-pair tiles use the chunked kernel");
  static_assert(!SPLIT || (!ROLL && N <= 64), "split mode: chunked kernel, segment sums in registers");
  constexpr int RK = kRows + K - 1;                  // halo rows one row block reads (per chunk)
  // rows are released as soon as their last tap row retired; !ROLL double-buffers chunks where that fits (K = 7: RK + 2)
  constexpr int kSlots = ROLL ? RK : (K == 7 ? RK + 2 : 2 * RK);
  constexpr int kPad = (K - 1) / 2, kPadW = (KW - 1) / 2;
  constexpr int F = N / 2;                           // accumulator registers per thread per output row
  constexpr int b_bytes = N * 128;
  constexpr int b_stride = (b_bytes + 1023) & ~1023;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* a_slots = smem;
  uint8_t* b_stages = smem + kSlots * kSlotBytes;
  const int kBStages = p.b_stages;
  uint64_t* bars = reinterpret_cast<uint64_t*>(b_stages + kBStages * b_stride);
  uint64_t* a_full = bars;                       // [kSlots]
  uint64_t* a_empty = a_full + kSlots;           // [kSlots]
  uint64_t* b_full = a_empty + kSlots;           // [kBStages]
  uint64_t* b_empty = b_full + kBStages;         // [kBStages]

  const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int strip = blockIdx.x % p.strips, rowblk = blockIdx.x / p.strips;
  constexpr int UPC = PK2 ? KW * RK : RK;          // halo units per (row block, chunk)
  const int n0 = blockIdx.y * N;
  const int img = PK2 ? 2 * blockIdx.z : blockIdx.z;
  const int x0 = strip * 128;
  const int NC = ROLL ? 1 : p.chunks;
  const int total_pairs = (p.H + kRows - 1) / kRows;
  const int pair0 = rowblk * p.pairs_per_cta;
  const int npairs = min(p.pairs_per_cta, total_pairs - pair0);
  const int y_base = pair0 * kRows;              // first output row of this CTA
  const int n_units = ROLL ? npairs * kRows + K - 1 : npairs * NC * UPC;

  if (threadIdx.x == 0) {
    for (int i = 0; i < kSlots; ++i) { mbar_init(a_full + i, 1); mbar_init(a_empty + i, kEmptyArrivals); }
    for (int i = 0; i < kBStages; ++i) { mbar_init(b_full + i, 1); mbar_init(b_empty + i, kEmptyArrivals); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  // everything above touched only this CTA's shared memory; the producing kernel's results are needed from here on
  asm volatile("griddepcontrol.wait;" ::: "memory");

  if (wg == 0) {
    // 384 threads start with 168 registers each; the producers need few, the consumers (2 rows x N/2 accumulators, the
    // split sums, the epilogue's packed outputs) many: 128 x 40 + 256 x 232 = 64 512 <= 65 536
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp == 0 && lane == 0) {
      // ===== halo-row producer =====
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_a)) : "memory");
      for (int u = 0; u < n_units; ++u) {
        const int slot = u % kSlots;
        const uint32_t round = static_cast<uint32_t>(u / kSlots);
        int ch = 0, yy, kw_p = 0;
        if (ROLL) {
          yy = y_base - kPad + u;
        } else {
          const int j = u / (NC * UPC), rem = u % (NC * UPC);
          ch = rem / UPC;
          kw_p = (rem % UPC) / RK;
          yy = y_base + j * kRows - kPad + rem % RK;
        }
        mbar_wait(a_empty + slot, (round & 1) ^ 1);
        const int a_ch = p.split ? (ch & 1) * p.cin_real + (ch >> 1) * 64 : ch * 64;  // split: chunk = (real chunk, hi | lo plane)
        if (PK2) {
          mbar_expect_tx(a_full + slot, static_cast<uint32_t>(2 * 64 * 128));
          tma_load_4d(a_slots + slot * kSlotBytes, &map_a, a_full + slot, a_ch, kw_p - kPadW, yy, img);
          tma_load_4d(a_slots + slot * kSlotBytes + 64 * 128, &map_a, a_full + slot, a_ch, kw_p - kPadW, yy, img + 1);
          continue;
        }
        mbar_expect_tx(a_full + slot, static_cast<uint32_t>((128 + KW - 1) * 128));
        tma_load_4d(a_slots + slot * kSlotBytes, &map_a, a_full + slot, a_ch, x0 - kPadW, yy, img);
      }
    } else if (warp == 1 && lane == 0) {
      // ===== weight producer =====
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_b)) : "memory");
      uint32_t it = 0;
      for (int j = 0; j < npairs; ++j)
        for (int ch = 0; ch < NC; ++ch) {
          // split: a hi chunk meets W_hi and W_lo (two tiles per tap), a lo chunk W_hi only; K-axis = [W_hi | W_lo | W_hi] per real chunk
          const int nrep = p.split && !(ch & 1) ? 2 : 1;
          for (int tap = 0; tap < K * KW; ++tap)
            for (int rep = 0; rep < nrep; ++rep, ++it) {
              const int st = it % kBStages;
              mbar_wait(b_empty + st, ((it / kBStages) & 1) ^ 1);
              mbar_expect_tx(b_full + st, static_cast<uint32_t>(b_bytes));
              const int kc = p.split ? (3 * (ch >> 1) + ((ch & 1) ? 2 : rep)) * 64 : ch * 64;
              const int tap_w = PK2 ? (tap % K) * K + tap / K : tap;  // PK2 consumes taps kw-major: (kw, kh) -> kh * K + kw
              tma_load_3d(b_stages + st * b_stride, &map_b, b_full + st, kc, n0, tap_w);
            }
        }
    }
    return;
  }

  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
  // ===== consumers: warpgroup g = wg - 1 owns tile rows (pixels) [64 g, 64 g + 64) =====
  const int g = wg - 1;
  const int m0 = 16 * (warp & 3) + (lane >> 2);    // this thread's accumulator rows: m0 and m0 + 8
  const int img_c = PK2 ? img + g : img;
  const int x_m0 = (PK2 ? 0 : x0 + 64 * g) + m0;
  // PK2: the second image's 64-pixel box sits 64 rows into the slot; otherwise pixel 64 g of the halo row is 64 g rows in
  const uint32_t a_base = smem_u32(a_slots) + static_cast<uint32_t>(g * 64 * 128), b_base = smem_u32(b_stages);
  const bool releaser = lane == 0;
  float acc[kRows][F];
  float accr[SPLIT ? kRows : 1][SPLIT ? F : 1];
  int st = 0;
  uint32_t b_phase = 0;
  int waited = 0;  // halo units whose TMA has been observed
  const int S = p.split ? p.seg_rows : K;
  for (int j = 0; j < npairs; ++j) {
#pragma unroll
    for (int r = 0; r < kRows; ++r)
#pragma unroll
      for (int i = 0; i < F; ++i) {
        acc[r][i] = 0.f;
        if (SPLIT) accr[r][i] = 0.f;
      }
    for (int ch = 0; ch < NC; ++ch)
    for (int kwo = 0; kwo < (PK2 ? KW : 1); ++kwo) {  // PK2: the kw shift is done by TMA, one set of halo rows per tap column
      const int base_u = ROLL ? j * kRows : PK2 ? ((j * NC + ch) * KW + kwo) * RK : (j * NC + ch) * RK;
      for (int kh = 0; kh < K; ++kh) {
        while (waited <= base_u + kh + kRows - 1 && waited < n_units) {
          mbar_wait(a_full + waited % kSlots, (waited / kSlots) & 1);
          ++waited;
        }
        uint32_t a_row[kRows];
#pragma unroll
        for (int r = 0; r < kRows; ++r) a_row[r] = a_base + ((base_u + r + kh) % kSlots) * kSlotBytes;
        const int nrep = p.split && !(ch & 1) ? 2 : 1;
        int prev_st = -1;
#pragma unroll
        for (int kw = 0; kw < (PK2 ? 1 : KW); ++kw)
        for (int rep = 0; rep < nrep; ++rep) {
          mbar_wait(b_full + st, b_phase);
          const uint32_t b_addr = b_base + st * b_stride;
          const uint32_t a_shift = PK2 ? 0u : static_cast<uint32_t>(kw * 128);
          wgmma_fence();
          // K step outer, row inner: consecutive MMAs go to different accumulators
#pragma unroll
          for (int k = 0; k < 4; ++k)
#pragma unroll
            for (int r = 0; r < kRows; ++r) wgmma(acc[r], make_desc(a_row[r] + a_shift + 32 * k), make_desc(b_addr + 32 * k));
          wgmma_commit();
          // keep one group in flight: the previous one has retired, so its weight stage goes back to the producer
          wgmma_wait<1>();
          if (prev_st >= 0 && releaser) mbar_arrive(b_empty + prev_st);
          prev_st = st;
          if (++st == kBStages) { st = 0; b_phase ^= 1; }
        }
        wgmma_wait<0>();
        fence_acc(acc);
        if (releaser) {
          mbar_arrive(b_empty + prev_st);
          // halo row base_u + kh is only read by tap rows <= kh of this block.  ROLL: rows >= kRows are also the next block's, so
          // only kh < kRows goes back to the producer now; !ROLL: every chunk fetches its own rows, so row kh is dead after tap row kh
          if (!ROLL || kh < kRows) mbar_arrive(a_empty + (base_u + kh) % kSlots);
        }
        if (SPLIT && (kh % S == S - 1 || kh == K - 1)) {
          // segment done: accumulate steps (tap rows) x KW x 4 K steps x (2 weight tiles for a hi chunk, 1 for a lo chunk).
          // The tensor core truncates each add towards zero: mean loss 0.36 x 2^-23 of the running sum per step (half an ulp,
          // ulp / |x| averaging 0.72 x 2^-23 over a binade), and a sum growing from 0 averages ~0.6 of its final value, so the
          // segment comes back short by ~0.216 x 2^-23 x m of itself: scaled back up here (leaves the zero-mean part).
          const int kh0 = (kh / S) * S;
          const int m_steps = min(S, K - kh0) * KW * 4 * ((ch & 1) ? 1 : 2);
          const float comp = 1.f + p.rz_comp * static_cast<float>(m_steps);
#pragma unroll
          for (int r = 0; r < kRows; ++r)
#pragma unroll
            for (int i = 0; i < F; ++i) {
              accr[r][i] = __fmaf_rn(acc[r][i], comp, accr[r][i]);
              acc[r][i] = 0.f;
            }
        }
      }
      if (releaser) {
        if (ROLL && K < kRows)  // fewer tap rows than output rows: release the rest of this block's own rows
          for (int i = K; i < kRows; ++i) mbar_arrive(a_empty + (base_u + i) % kSlots);
        if (!ROLL)  // the chunk's remaining halo rows (last read by tap row K - 1) are dead
          for (int i = K; i < RK; ++i) mbar_arrive(a_empty + (base_u + i) % kSlots);
      }
    }
    const int y0 = y_base + j * kRows;
    if (SPLIT) {
#pragma unroll
      for (int r = 0; r < kRows; ++r)
#pragma unroll
        for (int i = 0; i < F; ++i) acc[r][i] = __fmul_rn(accr[r][i], p.acc_scale);  // x 2^-s (exact)
    }
    epilogue_block<N>(p, cst, acc, img_c, y0, x_m0, n0, lane);
  }
}

// ---- host: tensor maps through the driver entry point (no -lcuda at link time)
using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                              const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                              CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeFn encode_fn() {
  static EncodeFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeFn>(p);
  });
  if (!fn) fail(SIVO_ECUDA, "cuTensorMapEncodeTiled is not available from this driver");
  return fn;
}

void encode(CUtensorMap* m, void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes, const cuuint32_t* box) {
  cuuint32_t elem[5] = {1, 1, 1, 1, 1};
  CUresult r = encode_fn()(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, rank, base, dims, strides_bytes, box, elem, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) fail(SIVO_ECUDA, "cuTensorMapEncodeTiled failed with %d", static_cast<int>(r));
}

}  // namespace

struct ConvTcPlan {
  CUtensorMap map_a, map_b;
  TcParams p;
  TcConsts cst;
  dim3 grid;
  size_t smem;
  int k;
  int kw;             // filter width the kernel walks (== k, or 1 for a window-folded layer)
  bool roll;
  bool pk2 = false;   // two images per 128-pixel M tile (layers at most 64 pixels wide, chunked 3x3 kernel)
  DevBuf w_own;       // weights the plan owns (the composed classifier)
};

namespace {
// one place that names every instantiation: configure == true sets the dynamic shared-memory limit, else launches
void conv_tc_dispatch(const ConvTcPlan& plan, cudaStream_t s, bool configure) {
  auto go = [&](auto kern) {
    // the limit is per kernel function, not per launch: always raise it to the full 227 KB so that plans of different
    // sizes that share an instantiation cannot lower it for each other
    if (configure) SIVO_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    else {
      // Programmatic dependent launch: the CTAs of this launch may start while the previous kernel of the stream is still
      // draining (on SMs it has already left, or never used) and run their prologue -- barrier init, descriptor
      // prefetch -- up to griddepcontrol.wait, which returns once that kernel has completed and flushed.  Opt-in
      // (SIVO_B200_PDL=1): the early CTAs sit on SMs the concurrent extractor kernels could have used.
      static const bool pdl = [] { const char* e = std::getenv("SIVO_B200_PDL"); return e && e[0] == '1'; }();
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = plan.grid;
      cfg.blockDim = dim3(kTcThreads);
      cfg.dynamicSmemBytes = plan.smem;
      cfg.stream = s;
      cudaLaunchAttribute attr[1];
      attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
      attr[0].val.programmaticStreamSerializationAllowed = 1;
      cfg.attrs = attr;
      cfg.numAttrs = pdl ? 1 : 0;
      SIVO_CUDA(cudaLaunchKernelEx(&cfg, kern, plan.map_a, plan.map_b, plan.p, plan.cst));
    }
  };
  // per (K, ROLL, KW, PK2): the three tile widths
  auto by_n = [&](auto k16, auto k64, auto k128) {
    if (plan.p.n_tile == 16) go(k16); else if (plan.p.n_tile == 64) go(k64); else go(k128);
  };
  const int K = plan.k;
  if (plan.p.split) {
    if (plan.p.n_tile == 16) { if (K == 7) go(k_conv_tc<7, false, 7, false, 16, true>); else if (K == 3) go(k_conv_tc<3, false, 3, false, 16, true>); else go(k_conv_tc<1, false, 1, false, 16, true>); }
    else { if (K == 7) go(k_conv_tc<7, false, 7, false, 64, true>); else if (K == 3) go(k_conv_tc<3, false, 3, false, 64, true>); else go(k_conv_tc<1, false, 1, false, 64, true>); }
  } else if (plan.kw == 1 && K > 1) {  // window-folded first layer (K x 1), 64-wide tiles
    if (K == 7) go(k_conv_tc<7, true, 1, false, 64, false>); else go(k_conv_tc<3, true, 1, false, 64, false>);
  } else if (plan.pk2) {
    if (plan.p.n_tile == 64) go(k_conv_tc<3, false, 3, true, 64, false>); else go(k_conv_tc<3, false, 3, true, 128, false>);
  } else if (plan.roll) {
    if (K == 7) by_n(k_conv_tc<7, true, 7, false, 16, false>, k_conv_tc<7, true, 7, false, 64, false>, k_conv_tc<7, true, 7, false, 128, false>);
    else if (K == 3) by_n(k_conv_tc<3, true, 3, false, 16, false>, k_conv_tc<3, true, 3, false, 64, false>, k_conv_tc<3, true, 3, false, 128, false>);
    else by_n(k_conv_tc<1, true, 1, false, 16, false>, k_conv_tc<1, true, 1, false, 64, false>, k_conv_tc<1, true, 1, false, 128, false>);
  } else {
    if (K == 7) by_n(k_conv_tc<7, false, 7, false, 16, false>, k_conv_tc<7, false, 7, false, 64, false>, k_conv_tc<7, false, 7, false, 128, false>);
    else if (K == 3) by_n(k_conv_tc<3, false, 3, false, 16, false>, k_conv_tc<3, false, 3, false, 64, false>, k_conv_tc<3, false, 3, false, 128, false>);
    else by_n(k_conv_tc<1, false, 1, false, 16, false>, k_conv_tc<1, false, 1, false, 64, false>, k_conv_tc<1, false, 1, false, 128, false>);
  }
}

int num_sms() {
  int dev = 0, n = 0;
  SIVO_CUDA(cudaGetDevice(&dev));
  SIVO_CUDA(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
  return std::max(1, n);
}
// Upper bound on the row blocks one CTA walks.  Long-lived CTAs amortise the prologue best, but while they run no SM
// frees up, so the extractors' short dependent kernels -- highest stream priority notwithstanding -- each wait for a
// whole CTA lifetime; SIVO_B200_TC_MAX_PPC trades the two (unit: 2-row blocks).
int tc_max_ppc() {
  static const int v = [] { const char* e = std::getenv("SIVO_B200_TC_MAX_PPC"); return e ? std::max(1, atoi(e)) : 48; }();
  return v;
}
size_t tc_smem_bytes(int K, bool roll, int n_tile, int stages) {
  const int rk = kRows + K - 1;
  const int slots = roll ? rk : (K == 7 ? rk + 2 : 2 * rk);  // k_conv_tc's kSlots
  const int b_stride = (n_tile * 128 + 1023) & ~1023;
  return 1024 + static_cast<size_t>(slots) * kSlotBytes + static_cast<size_t>(stages) * b_stride + (2 * slots + 2 * stages) * 8;
}
int tc_stages(int K, bool roll, int n_tile) {  // deepest weight ring that fits (0 = configuration does not fit)
  for (int st = kMaxBStages; st >= 3; --st)
    if (tc_smem_bytes(K, roll, n_tile, st) <= 227 * 1024) return st;
  return 0;
}
int tc_pick_n(const Op& op, const TensorView& out, bool roll) {
  if (out.dt == DType::F32 && out.cs <= 16) return 16;  // the float logits layer
  if (op.split || op.fold_kw) return 64;                // split: the segment sums must fit in registers next to the accumulators
  int n = (op.cout_p % 128 == 0) ? 128 : 64;
  if (!tc_stages(op.k, roll, n)) n = 64;
  return n;
}
// row blocks per CTA: minimise (waves over the SMs) x (blocks per CTA + ~1 block of prologue / halo overhead)
int tc_blocks_per_cta(long columns, int total_pairs, double overhead) {
  const int sms = num_sms();
  int ppc = 1;
  double best_cost = 1e30;
  for (int c = 1; c <= std::min(total_pairs, tc_max_ppc()); ++c) {
    const long ctas = columns * ceil_div(total_pairs, c);
    const double cost = static_cast<double>((ctas + sms - 1) / sms) * (c + overhead);
    if (cost < best_cost - 1e-9) { best_cost = cost; ppc = c; }
  }
  return ppc;
}
}  // namespace

bool conv_tc_supported(const Op& op, const TensorView& in, const TensorView& out) {
  if (const char* e = std::getenv("SIVO_B200_NO_TC")) if (e[0] == '1') return false;
  if (in.dt != DType::F16) return false;
  if (op.k != 1 && op.k != 3 && op.k != 7) return false;
  if (op.cout_p > kMaxCout) return false;
  if (op.fold_kw) {
    if (in.cs != 8 || op.cin_p != 64 || (op.k != 3 && op.k != 7) || out.dt != DType::F16 || op.cout % 64 || out.cs != op.cout) return false;
    return tc_stages(op.k, true, tc_pick_n(op, out, true)) > 0;
  }
  if (op.split) {  // `in` = the [hi Cin | lo Cin] half planes of the float input
    if (op.cin % 64 || in.cs != 2 * op.cin || out.dt != DType::F32) return false;
    if (!((out.cs == op.cout && op.cout % 64 == 0) || (out.cs == 16 && op.cout <= 16))) return false;
    return tc_stages(op.k, false, tc_pick_n(op, out, false)) > 0;
  }
  if (in.cs % 64 || op.cin != in.cs) return false;
  if (out.dt == DType::F16) {
    if (op.cout % 64 || out.cs != op.cout) return false;
  } else {
    if (out.cs != 16 || op.cout > 16) return false;  // float logits, 16-channel pixels
  }
  const bool roll = in.cs == 64;
  return tc_stages(op.k, roll, tc_pick_n(op, out, roll)) > 0;
}

std::shared_ptr<ConvTcPlan> conv_tc_plan(const Op& op, const TensorView& in, const TensorView& out, const void* w_tc) {
  auto plan = std::make_shared<ConvTcPlan>();
  const int K = op.k;
  const int KW = op.fold_kw ? 1 : K;
  const bool roll = (in.cs == 64 || op.fold_kw) && !op.split;
  const int n_tile = tc_pick_n(op, out, roll);
  if (op.fold_kw) {
    // window-folded input: `in` is the zero-padded 8-channel image [N][H][W + 8][8] half (3 zero pixels left, 5 right);
    // "pixel" x of the operand is the 128-byte window of 8 pixels x 8 channels starting at padded pixel x, i.e. image
    // pixels x-3 .. x+4: a tensor whose W stride (16 B) is smaller than its row (128 B).  TMA only needs 16-byte
    // multiples, so one box {64, 128, 1, 1} lands the K = kw*8 + c operand rows of 128 output pixels, and the K x K
    // layer over 3 channels becomes a K x 1 layer over these 64 -- no expanded tensor in HBM.  `in.w` counts the padded row.
    const int w_valid = in.w - 8;
    cuuint64_t dims[4] = {64, static_cast<cuuint64_t>(w_valid), static_cast<cuuint64_t>(in.h), static_cast<cuuint64_t>(in.n)};
    cuuint64_t strides[3] = {16, static_cast<cuuint64_t>(in.w) * 16, static_cast<cuuint64_t>(in.h) * in.w * 16};
    cuuint32_t box[4] = {64, 128, 1, 1};
    encode(&plan->map_a, in.p, 4, dims, strides, box);
  } else {  // input: NHWC half, dims (C, W, H, N)
    cuuint64_t dims[4] = {static_cast<cuuint64_t>(in.cs), static_cast<cuuint64_t>(in.w), static_cast<cuuint64_t>(in.h),
                          static_cast<cuuint64_t>(in.n)};
    cuuint64_t strides[3] = {static_cast<cuuint64_t>(in.cs) * 2, static_cast<cuuint64_t>(in.w) * in.cs * 2,
                             static_cast<cuuint64_t>(in.h) * in.w * in.cs * 2};
    plan->pk2 = !roll && !op.split && K == 3 && in.w <= 64 && in.n >= 2 && n_tile != 16;
    cuuint32_t box[4] = {64, static_cast<cuuint32_t>(plan->pk2 ? 64 : 128 + K - 1), 1, 1};
    encode(&plan->map_a, in.p, 4, dims, strides, box);
  }
  {  // weights: [tap][cout_p][cin_p] half, dims (cin, cout, tap)
    const int kext = op.split ? 3 * op.cin_p : op.cin_p;  // split: [W_hi | W_lo | W_hi] per 64-channel chunk along K
    cuuint64_t dims[3] = {static_cast<cuuint64_t>(kext), static_cast<cuuint64_t>(op.cout_p), static_cast<cuuint64_t>(K * KW)};
    cuuint64_t strides[2] = {static_cast<cuuint64_t>(kext) * 2, static_cast<cuuint64_t>(op.cout_p) * kext * 2};
    cuuint32_t box[3] = {64, static_cast<cuuint32_t>(n_tile), 1};
    encode(&plan->map_b, const_cast<void*>(w_tc), 3, dims, strides, box);
  }
  TcParams& p = plan->p;
  p.H = in.h; p.W = op.fold_kw ? in.w - 8 : in.w; p.N_batch = in.n;
  p.cout_total = out.cs;
  p.n_tile = n_tile;
  p.chunks = op.fold_kw ? 1 : in.cs / 64;
  p.out_f32 = out.dt == DType::F32 ? (n_tile == 16 ? 1 : 2) : 0;
  p.split = op.split ? 1 : 0;
  p.cin_real = op.cin;
  p.acc_scale = op.split ? op.acc_scale : 1.f;
  p.seg_rows = 1;  // a segment per (chunk, tap row): 7x7 56 / 28 accumulate steps, 3x3 24 / 12, 1x1 8 / 4
  if (const char* e = std::getenv("SIVO_B200_SPLIT_SEG")) p.seg_rows = std::max(1, std::min(K, atoi(e)));
  p.rz_comp = 0.216f * 1.1920929e-7f;  // x 2^-23
  if (const char* e = std::getenv("SIVO_B200_SPLIT_RZ")) p.rz_comp = static_cast<float>(atof(e)) * 1.1920929e-7f;
  p.strips = ceil_div(p.W, 128);
  const int cout_tiles = p.out_f32 == 1 ? 1 : op.cout_p / n_tile;
  const int n_z = plan->pk2 ? ceil_div(in.n, 2) : in.n;  // PK2: an image pair per tile
  const int columns = p.strips * n_z * cout_tiles;
  const int total_pairs = ceil_div(in.h, kRows);
  p.pairs_per_cta = tc_blocks_per_cta(columns, total_pairs, roll ? (K - 1.0) / kRows * 0.5 + 0.5 : 0.3);
  p.relu = op.relu; p.has_bn = op.has_bn; p.slope = op.slope;
  std::memset(&plan->cst, 0, sizeof(TcConsts));
  if (static_cast<int>(op.h_bias.size()) != op.cout_p || (op.has_bn && (static_cast<int>(op.h_bn_scale.size()) != op.cout_p ||
                                                                         static_cast<int>(op.h_bn_shift.size()) != op.cout_p)))
    fail(SIVO_EINVAL, "conv_tc_plan: host copies of the bias / BN constants are missing");
  std::copy(op.h_bias.begin(), op.h_bias.end(), plan->cst.bias);
  if (op.has_bn) {
    std::copy(op.h_bn_scale.begin(), op.h_bn_scale.end(), plan->cst.bn_scale);
    std::copy(op.h_bn_shift.begin(), op.h_bn_shift.end(), plan->cst.bn_shift);
  }
  p.out = out.p;
  p.has_drop = 0; p.seed = 0; p.frame = nullptr; p.drop_layer = 0; p.drop_scale = 2.f;
  p.unpool_mask = nullptr; p.mask_n = 1;
  p.pool_out = nullptr; p.pool_mask = nullptr;
  p.has_cls = 0; p.cls_out = nullptr;
  plan->grid = dim3(p.strips * ceil_div(total_pairs, p.pairs_per_cta), cout_tiles, n_z);
  p.b_stages = tc_stages(K, roll, n_tile);
  plan->smem = tc_smem_bytes(K, roll, n_tile, p.b_stages);
  plan->k = K;
  plan->kw = KW;
  plan->roll = roll;
  conv_tc_dispatch(*plan, nullptr, true);
  return plan;
}

void conv_tc_set_dropout(ConvTcPlan& plan, uint64_t seed, const uint64_t* frame_dev, int layer, float scale) {
  plan.p.has_drop = 1;
  plan.p.seed = seed;
  plan.p.frame = frame_dev;
  plan.p.drop_layer = layer;
  plan.p.drop_scale = scale;
}

void conv_tc_set_unpool(ConvTcPlan& plan, const uint8_t* mask, int mask_n, void* out_2h_2w) {
  plan.p.unpool_mask = mask;
  plan.p.mask_n = mask_n;
  plan.p.out = out_2h_2w;
}

std::vector<__half> conv_tc_split_weights(const float* W, int cout, int cin, int K, int cout_p, int cin_p, float* acc_scale) {
  // [tap][cout_p][3 cin_p] half: per 64-channel chunk c of the K axis [W_hi(c) | W_lo(c) | W_hi(c)], where W * 2^s = W_hi + W_lo.
  // The power-of-two scale lifts the low parts out of half's subnormal range (|w| ~ 1e-2 has ulp(hi) ~ 2^-17 < 2^-14); the
  // epilogue multiplies the accumulator by 2^-s, which is exact.
  float wmax = 0.f;
  for (size_t i = 0; i < static_cast<size_t>(cout) * cin * K * K; ++i) wmax = std::max(wmax, std::fabs(W[i]));
  int e = 0;
  if (wmax > 0.f && std::isfinite(wmax)) { std::frexp(wmax, &e); e = 8 - e; }  // wmax * 2^e in [128, 256)
  e = std::max(-24, std::min(24, e));
  const float up = std::ldexp(1.f, e);
  *acc_scale = std::ldexp(1.f, -e);
  const int kext = 3 * cin_p;
  std::vector<__half> wt(static_cast<size_t>(K) * K * cout_p * kext, __float2half_rn(0.f));
  for (int co = 0; co < cout; ++co)
    for (int ci = 0; ci < cin; ++ci)
      for (int t = 0; t < K * K; ++t) {
        const float v = W[(static_cast<size_t>(co) * cin + ci) * K * K + t] * up;
        const __half hi = __float2half_rn(v), lo = __float2half_rn(v - __half2float(hi));
        __half* row = wt.data() + (static_cast<size_t>(t) * cout_p + co) * kext + (ci / 64) * 192 + ci % 64;
        row[0] = hi; row[64] = lo; row[128] = hi;
      }
  return wt;
}

bool conv_tc_can_fuse_pool(const ConvTcPlan& plan) {
  return !plan.p.out_f32 && !plan.p.unpool_mask && !plan.p.has_drop && !plan.p.has_cls && (plan.p.H % 2) == 0 && (plan.p.W % 2) == 0;
}

void conv_tc_set_pool(ConvTcPlan& plan, void* pooled, uint8_t* mask) {
  plan.p.pool_out = static_cast<__half*>(pooled);
  plan.p.pool_mask = mask;
}

bool conv_tc_can_fuse_classifier(const ConvTcPlan& plan) {
  return plan.roll && plan.p.n_tile == 64 && plan.p.cout_total == 64 && !plan.p.out_f32 && !plan.p.unpool_mask && !plan.p.has_drop && !plan.p.pool_out;
}

void conv_tc_set_classifier(ConvTcPlan& plan, const float* w_cin_by_cout, int stride, const float* bias, int n_bias, float* logits) {
  for (int c = 0; c < 64; ++c)
    for (int j = 0; j < 16; ++j) plan.cst.cls_w[c * 16 + j] = j < stride ? w_cin_by_cout[static_cast<size_t>(c) * stride + j] : 0.f;
  for (int j = 0; j < 16; ++j) plan.cst.cls_b[j] = j < n_bias ? bias[j] : 0.f;
  plan.p.has_cls = 1;
  plan.p.cls_out = logits;
}

bool conv_tc_can_compose_classifier(const ConvTcPlan& plan) {
  return plan.roll && plan.k == 7 && plan.kw == 7 && plan.p.n_tile == 64 && !plan.p.out_f32 && !plan.p.unpool_mask &&
         !plan.p.has_drop && !plan.p.pool_out && !plan.p.has_cls && !plan.p.relu && !plan.p.has_bn && plan.p.cout_total == 64;
}

void conv_tc_set_composed_classifier(ConvTcPlan& plan, const Op& conv, const float* wc, const float* bc, int n_cls, float* logits) {
  const int K = 7;
  if (n_cls > 16 || conv.h_w_raw.size() != static_cast<size_t>(64) * 64 * K * K || conv.h_bias.size() < 64)
    fail(SIVO_EINVAL, "composed classifier: unexpected layer shapes");
  // W'[o][i][kh][kw] = sum_c wc[o][c] W[c][i][kh][kw] in double, rounded once to half; rows o >= n_cls stay zero.
  // Device layout [kh][kw][16][64]: the [tap][cout][cin] layout of every other weight tensor, 16-row tiles.
  std::vector<__half> w(static_cast<size_t>(K) * K * 16 * 64, __float2half_rn(0.f));
  const float* W = conv.h_w_raw.data();
  for (int o = 0; o < n_cls; ++o)
    for (int i = 0; i < 64; ++i)
      for (int kh = 0; kh < K; ++kh)
        for (int kw = 0; kw < K; ++kw) {
          double acc = 0.0;
          for (int c = 0; c < 64; ++c) acc += static_cast<double>(wc[o * 64 + c]) * W[((static_cast<size_t>(c) * 64 + i) * K + kh) * K + kw];
          w[((static_cast<size_t>(kh) * K + kw) * 16 + o) * 64 + i] = __float2half_rn(static_cast<float>(acc));
        }
  plan.w_own.alloc(w.size() * sizeof(__half));
  SIVO_CUDA(cudaMemcpy(plan.w_own.p, w.data(), w.size() * sizeof(__half), cudaMemcpyHostToDevice));
  cuuint64_t dims[3] = {64, 16, static_cast<cuuint64_t>(K) * K};
  cuuint64_t strides[2] = {128, 16 * 128};
  cuuint32_t box[3] = {64, 16, 1};
  encode(&plan.map_b, plan.w_own.p, 3, dims, strides, box);
  std::memset(&plan.cst, 0, sizeof(TcConsts));
  for (int o = 0; o < n_cls; ++o) {
    double acc = bc[o];
    for (int c = 0; c < 64; ++c) acc += static_cast<double>(wc[o * 64 + c]) * conv.h_bias[c];
    plan.cst.bias[o] = static_cast<float>(acc);
  }
  TcParams& p = plan.p;
  p.out_f32 = 1;
  p.n_tile = 16;
  p.cout_total = 16;
  p.out = logits;
  p.b_stages = tc_stages(K, true, 16);
  plan.smem = tc_smem_bytes(K, true, 16, p.b_stages);
  plan.grid.y = 1;
  conv_tc_dispatch(plan, nullptr, true);
}

void conv_tc_launch(const ConvTcPlan& plan, const Op& op, cudaStream_t s) {
  (void)op;
  conv_tc_dispatch(plan, s, false);
  SIVO_CUDA(cudaGetLastError());
}

}  // namespace sivo
