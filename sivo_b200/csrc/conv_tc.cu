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
//    affine / ReLU -> half, then store | dropout | max-unpool scatter | 2x2 max-pool + argmax, or -> float logits.  Both
//    consumers read every weight stage, so they reach a block's epilogue together and no MMA is issued while it runs.
//    The 64-wide store / dropout / unpool epilogues are therefore deferred: a block's outputs are converted and staged in
//    registers (16 B per lane after a quad transpose), and their stores are issued one slice per tap row between the next
//    block's MMA commits, so they drain under the tensor core's work.
//  * Constants (bias, BN) are kernel parameters: the epilogue reads them from the constant bank and leaves the
//    shared-memory data path to the MMA operand reads.
//  * The Cin = 64, 7x7 layers with 64-wide half output tiles (Basic's conv1 .. conv_decode2) run on k_conv_tn instead: the
//    same producers and rings with the GEMM transposed -- the weights as M, all 128 pixels of a row as N -- and an
//    epilogue staged through shared memory.  Fed by a max-unpool (Basic's decoder), it unpools as it loads its halo rows.
//  * The 64 -> 16 float-logits layers (K = 3, 7) run on k_conv_stack instead: tap rows stacked along N, resident weights.
//    Fed by a max-unpool (Basic's composed classifier), it unpools the pooled tensor as it loads its halo rows.
#include <cuda.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <type_traits>
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
  int rows_per_cta;        // k_conv_stack: output rows one CTA emits, a piece of the flattened (image, strip, row) range
  int strips;              // ceil(W / 128)
  int relu, has_bn, has_drop;
  float slope;
  void* out;
  // dropout fused into the epilogue (decoder convs of Basic: decdrop4 / decdrop3)
  uint64_t seed;
  const uint64_t* frame;
  uint32_t drop_nl;        // sample0 | layer << 16: local image i draws the keep bits of dropout layer `layer`, global sample
                           // sample0 + i (a shard handle owns samples [sample0, sample0 + N_batch) of the frame)
  float drop_scale;
  // max-unpool fused into the epilogue (decoder convs): the output tensor is 2H x 2W and every pixel's channel
  // lands in the 2x2 position its pooling mask names, zeros elsewhere (upsample_layer.cpp:74-103)
  const uint8_t* unpool_mask;
  int mask_n;
  // 2x2/2 max pool with argmax fused into the epilogue (encoder convs): only the pooled tensor and its 2-bit mask are
  // written (pooling_layer.cpp:140-187: scan (0,0),(0,1),(1,0),(1,1), strict '>', so the first maximum wins)
  __half* pool_out;        // [N][H/2][W/2][cout_total]
  uint8_t* pool_mask;      // same shape
  // k_conv_stack<K, true>, k_conv_tn<7, 7, true>: the input is the max-unpool of this pooled tensor [N][H/2][W/2][64] by
  // unpool_mask (same shape, batch mask_n), expanded as the halo rows are loaded; the H x W unpooled tensor is never
  // stored, and the epilogue does not scatter (unpool_mask is the input's)
  const __half* unpool_in;
};

// Per-layer constants, passed by value as a kernel parameter so that the epilogue reads them from the constant bank.
constexpr int kMaxCout = 512;
struct TcConsts {
  float bias[kMaxCout], bn_scale[kMaxCout], bn_shift[kMaxCout];
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
// k_conv_stack's MMA: D[64 x 16 K] += A[64 x 16] * B[16 x 16 K], column block j into ring slot acc[j].  The slots keep fixed
// registers: HGMMA takes its accumulators as one register range, and ptxas serialises every wgmma of a kernel whose MMAs
// name different sub-ranges or orders of the same registers.
#define SIVO_ACC8(s) "+f"(acc[s][0]), "+f"(acc[s][1]), "+f"(acc[s][2]), "+f"(acc[s][3]), "+f"(acc[s][4]), "+f"(acc[s][5]), \
                     "+f"(acc[s][6]), "+f"(acc[s][7])
__device__ __forceinline__ void wgmma_stack(float (&acc)[7][8], uint64_t a, uint64_t b) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n112k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, "
      "%47, %48, %49, %50, %51, %52, %53, %54, %55}, %56, %57, 1, 1, 1, 0, 0;"
      : SIVO_ACC8(0), SIVO_ACC8(1), SIVO_ACC8(2), SIVO_ACC8(3), SIVO_ACC8(4), SIVO_ACC8(5), SIVO_ACC8(6)
      : "l"(a), "l"(b));
}
__device__ __forceinline__ void wgmma_stack(float (&acc)[3][8], uint64_t a, uint64_t b) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, "
      "%24, %25, 1, 1, 1, 0, 0;"
      : SIVO_ACC8(0), SIVO_ACC8(1), SIVO_ACC8(2)
      : "l"(a), "l"(b));
}
#undef SIVO_ACC8
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Ties the accumulator registers to the preceding wait: the compiler must not move their reads (or the zeroing of a
// fresh segment) across it.  Takes a register array of any rank.
template <typename T, int F>
__device__ __forceinline__ void fence_acc(T (&d)[F]) {
#pragma unroll
  for (int i = 0; i < F; ++i) {
    if constexpr (std::is_array_v<T>) fence_acc(d[i]);
    else asm volatile("" : "+f"(d[i])::"memory");
  }
}

// One of four words by a run-time index: selects, not a dynamically indexed (= local-memory) array.
__device__ __forceinline__ uint32_t pick4(const uint32_t (&a)[4], int i) { return i == 0 ? a[0] : i == 1 ? a[1] : i == 2 ? a[2] : a[3]; }

// Dropout on two channels' half values in one word: y = x * keep * scale (exact), keep = bits `bit`, `bit` + 1 of `keep`.
__device__ __forceinline__ uint32_t drop_word(uint32_t w, uint32_t keep, int bit, float scale) {
  __half2 hv = *reinterpret_cast<const __half2*>(&w);
  hv = __hmul2(hv, __floats2half2_rn((keep >> bit) & 1u ? scale : 0.f, (keep >> (bit + 1)) & 1u ? scale : 0.f));
  return *reinterpret_cast<const uint32_t*>(&hv);
}

// 2x2 max-pool of two channels' half values per word over a window in scan order: a = (y, x), b = (y, x+1), c = (y+1, x),
// d = (y+1, x+1).  Strict '>' per half (false on NaN, like __hgt), so the first maximum wins; `arg` gets its position
// (0 .. 3) in bytes 0 and 1.
__device__ __forceinline__ uint32_t pool2x2(uint32_t a, uint32_t b, uint32_t c, uint32_t d, uint32_t& arg) {
  uint32_t best = a;
  arg = 0;
  const uint32_t cand[3] = {b, c, d};
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const uint32_t sel = __hgt2_mask(*reinterpret_cast<const __half2*>(&cand[k]), *reinterpret_cast<const __half2*>(&best));  // 0xFFFF where the candidate wins
    best = (best & ~sel) | (cand[k] & sel);
    const uint32_t selb = __byte_perm(sel, 0u, 0x4420);  // the two half masks as two byte masks (bytes 0 and 1)
    arg = (arg & ~selb) | ((0x0101u * static_cast<uint32_t>(k + 1)) & selb);
  }
  return best;
}

__device__ __forceinline__ float affine(const TcParams& p, const TcConsts& cst, float v, int c) {
  float t = __fadd_rn(v, cst.bias[c]);
  if (p.has_bn) t = __fadd_rn(__fmul_rn(t, cst.bn_scale[c]), cst.bn_shift[c]);
  // a negative input gives +0 (Caffe's max(t, 0) + slope * min(t, 0)), not slope * t = -0
  if (p.relu) t = t > 0.f ? t : (p.slope != 0.f ? __fmul_rn(p.slope, t) : 0.f);
  return t;
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
        uint32_t arg;
        const uint32_t best = pool2x2(a, b, cc, d, arg);
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
        dropout_bits128_nl(p.seed, *p.frame, p.drop_nl + img, static_cast<uint32_t>(y * p.W + x), n0 >> 7, bits);
      const size_t mask_pix = (static_cast<size_t>(img % p.mask_n) * p.H + y) * p.W + x;
#pragma unroll
      for (int j = 0; j < N / 8; ++j) {
        const int c = n0 + 8 * j + 2 * q;
        const __half2 hv = __floats2half2_rn(affine(p, cst, acc[r][4 * j + 2 * h], c), affine(p, cst, acc[r][4 * j + 2 * h + 1], c + 1));
        uint32_t w = *reinterpret_cast<const uint32_t*>(&hv);
        if (p.has_drop) w = drop_word(w, pick4(bits, (c >> 5) & 3), c & 31, p.drop_scale);
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

// Deferred epilogue (store / dropout / max-unpool, N = 64): the half outputs of one row block, staged in registers so that
// their stores can be issued while the next row block's MMAs run.  Chunk i = (2 r + h) * N/32 + J holds channels
// 8 (4 J + q) .. + 7 of pixel (y0 + r, x_m0 + 8 h): 16 bytes per lane, 64 contiguous bytes per quad.
template <int N>
struct EpiStage {
  static constexpr int kChunks = kRows * 2 * (N / 32);
  uint4 v[kChunks];
  uint2 m[kChunks];  // unpool: the chunk's 8 mask bytes
  int y0, img;
};

// 4 x 4 word transpose within a quad: lane q holds w[k] = channels 8 k + 2 q, +1 of a 32-channel group and gets back
// channels 8 q .. 8 q + 7 (lane q' sends w[q' ^ x] across xor distance x, which is the word lane q' ^ x keeps).
__device__ __forceinline__ uint4 quad_transpose(const uint32_t (&w)[4], int q) {
  uint32_t r[4];  // r[x] = word q of column q ^ x
  r[0] = pick4(w, q);
#pragma unroll
  for (int x = 1; x < 4; ++x) r[x] = __shfl_xor_sync(0xffffffffu, pick4(w, q ^ x), x);
  return make_uint4(pick4(r, q), pick4(r, q ^ 1), pick4(r, q ^ 2), pick4(r, q ^ 3));
}

// Converts one row block's accumulators into its staged outputs with the arithmetic of epilogue_block (bias / BN /
// ReLU -> half, dropout keep bits x scale) and issues the unpool mask loads.  Called by all 32 lanes (warp shuffles).
template <int N>
__device__ __forceinline__ void epilogue_stage(const TcParams& p, const TcConsts& cst, const float (&acc)[kRows][N / 2], int img,
                                               int y0, int x_m0, int n0, int q, EpiStage<N>& e) {
  e.y0 = y0;
  e.img = img;
  const bool img_ok = img < p.N_batch;
#pragma unroll
  for (int r = 0; r < kRows; ++r) {
    const int y = y0 + r;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int x = x_m0 + 8 * h;
      const bool inside = y < p.H && img_ok && x < p.W;
      uint32_t bits[4] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu};
      if (p.has_drop && inside)
        dropout_bits128_nl(p.seed, *p.frame, p.drop_nl + img, static_cast<uint32_t>(y * p.W + x), n0 >> 7, bits);
      uint32_t w[N / 8];
#pragma unroll
      for (int j = 0; j < N / 8; ++j) {
        const int c = n0 + 8 * j + 2 * q;
        const __half2 hv = __floats2half2_rn(affine(p, cst, acc[r][4 * j + 2 * h], c), affine(p, cst, acc[r][4 * j + 2 * h + 1], c + 1));
        w[j] = *reinterpret_cast<const uint32_t*>(&hv);
        if (p.has_drop) w[j] = drop_word(w[j], pick4(bits, (c >> 5) & 3), c & 31, p.drop_scale);
      }
      const size_t mask_pix = (static_cast<size_t>(img % p.mask_n) * p.H + y) * p.W + x;
#pragma unroll
      for (int J = 0; J < N / 32; ++J) {
        const int i = (2 * r + h) * (N / 32) + J;
        const uint32_t wj[4] = {w[4 * J], w[4 * J + 1], w[4 * J + 2], w[4 * J + 3]};
        e.v[i] = quad_transpose(wj, q);
        e.m[i] = make_uint2(0u, 0u);
        if (p.unpool_mask && inside)
          e.m[i] = __ldg(reinterpret_cast<const uint2*>(p.unpool_mask + mask_pix * p.cout_total + n0 + 8 * (4 * J + q)));
      }
    }
  }
}

// The max-unpool scatter of 8 channels (16 bytes `v`) of pixel (y, x): each channel's value goes to the 2x2 position of the
// 2H x 2W output its mask byte (of `m`) names, zeros to the other three.
__device__ __forceinline__ void unpool_store8(const TcParams& p, int img, int y, int x, int c, uint4 v, uint2 m) {
  __half* const ob = static_cast<__half*>(p.out) + ((static_cast<size_t>(img) * 2 * p.H + 2 * y) * (2 * p.W) + 2 * x) * p.cout_total + c;
  const size_t row_step = static_cast<size_t>(2 * p.W) * p.cout_total;
#pragma unroll
  for (int pos = 0; pos < 4; ++pos) {
    const uint32_t lo = __vcmpeq4(m.x, 0x01010101u * pos), hi = __vcmpeq4(m.y, 0x01010101u * pos);  // 0xFF per matching byte
    const uint4 o = make_uint4(v.x & __byte_perm(lo, 0u, 0x1100), v.y & __byte_perm(lo, 0u, 0x3322),
                               v.z & __byte_perm(hi, 0u, 0x1100), v.w & __byte_perm(hi, 0u, 0x3322));
    *reinterpret_cast<uint4*>(ob + (pos >> 1) * row_step + (pos & 1) * p.cout_total) = o;
  }
}

// Issues the stores of staged chunk i (a compile-time index after unrolling): one 16-byte store, or four for unpool.
template <int N>
__device__ __forceinline__ void epilogue_flush(const TcParams& p, const EpiStage<N>& e, int i, int x_m0, int n0, int q) {
  const int r = i / (2 * (N / 32)), h = (i / (N / 32)) & 1, J = i % (N / 32);
  // opaque copies: the addresses are computed here, not at staging time and kept live (in spilled registers) across the MMAs
  int y0 = e.y0, img = e.img;
  asm volatile("" : "+r"(y0), "+r"(img));
  const int y = y0 + r, x = x_m0 + 8 * h;
  if (!(y < p.H && img < p.N_batch && x < p.W)) return;
  const int c = n0 + 8 * (4 * J + q);
  const uint4 v = e.v[i];
  if (p.unpool_mask) {
    unpool_store8(p, img, y, x, c, v, e.m[i]);
  } else {
    *reinterpret_cast<uint4*>(static_cast<__half*>(p.out) + ((static_cast<size_t>(img) * p.H + y) * p.W + x) * p.cout_total + c) = v;
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
//
// TcCta's shared memory, in this order: the halo ring (tc_slots rows of kSlotBytes), the weight ring (`stages` tiles of
// N couts x 64 cin half, each 1 KB aligned), `stage_bytes` for the consumers' epilogue staging, then the full / empty
// mbarriers of both rings; the leading 1 KB aligns the dynamic shared-memory base.
__host__ __device__ constexpr int tc_slots(int K, bool roll) {
  // rows are released as soon as their last tap row retired; !ROLL double-buffers chunks where that fits (K = 7: RK + 2)
  return roll ? kRows + K - 1 : (K == 7 ? kRows + K + 1 : 2 * (kRows + K - 1));
}
__host__ __device__ constexpr int tc_b_stride(int n) { return (n * 128 + 1023) & ~1023; }
__host__ __device__ constexpr int tc_smem_bytes(int K, bool roll, int n, int stages, int stage_bytes) {
  return 1024 + tc_slots(K, roll) * kSlotBytes + stages * tc_b_stride(n) + stage_bytes + (2 * tc_slots(K, roll) + 2 * stages) * 8;
}
// the deepest weight ring that fits (0: none of at least 3 stages does)
__host__ __device__ constexpr int tc_stages(int K, bool roll, int n, int stage_bytes) {
  for (int st = kMaxBStages; st >= 3; --st)
    if (tc_smem_bytes(K, roll, n, st, stage_bytes) <= 227 * 1024) return st;
  return 0;
}

// The halo-row producer of a convolution whose input is a max-unpool (k_conv_stack<K, true>, k_conv_tn<K, K, true>), run
// by NT threads of warpgroup 0: each halo row -- input row y of the H x W unpooled tensor, pixels x0 - pad .. x0 + 127 + pad
// -- is expanded from pooled row y / 2 straight into its ring slot.  Per pooled pixel j and 8-channel chunk c, one thread
// loads the 16 bytes of values and the 8 mask bytes and writes the 16-byte chunks of pixels 2 j and 2 j + 1: each channel
// keeps its value where its mask code is 2 (y & 1) + dx and is zero elsewhere, the select the unpool kernel makes, so the
// slot holds the bits the unpooled tensor would.  Chunks go to their SWIZZLE_128B position (the slots are 1 KB aligned);
// rows and pixels outside the image are written as zeros, since slots are reused (TMA's zero fill in the plain kernels).
// A row's loads are issued before the wait for its slot, so their latency hides under the consumers' MMAs of the
// previous row.
template <int K, int NT>
struct HaloUnpool {
  static constexpr int kPad = (K - 1) / 2;
  static constexpr int kHalo = 128 + K - 1;
  static constexpr int kLeft = (kPad + 1) / 2;                  // pooled pixels the halo reaches left of x0 / 2
  static constexpr int kPooled = kLeft + (127 + kPad) / 2 + 1;  // pooled pixels per halo row (68 for K = 7)
  static constexpr int kJStep = NT / 8;                         // pooled pixels between a thread's consecutive steps
  static constexpr int kSteps = (kPooled + kJStep - 1) / kJStep;  // (pixel, chunk) pairs per thread
  static_assert(NT % 32 == 0 && kJStep % 4 == 0, "whole warps; steps 2 kJStep pixels apart keep the swizzle phase");
  // thread tid: chunk c of pooled pixels j = jt + kJStep s (halo-relative jr = jr0 + kJStep s); the addresses of steps s
  // differ by compile-time strides, so a row needs one pointer per tensor
  const int c, jr0;
  const int px0;  // halo pixel of (jr0, dx = 0): image pixel x0 - pad + px = 2 j + dx.  Its swizzle phase px & 7 is the same for every step.
  int jt = 0;
  uint32_t live = 0;  // steps whose pooled pixel is inside the image
  long v_img = 0, m_img = 0;

  __device__ __forceinline__ explicit HaloUnpool(int tid) : c(tid & 7), jr0(tid >> 3), px0(2 * (tid >> 3) + kPad - 2 * kLeft) {}

  // the strip starting at pixel x0 of image img
  __device__ __forceinline__ void strip(const TcParams& p, int img, int x0) {
    const int Hp = p.H >> 1, Wp = p.W >> 1;
    jt = (x0 >> 1) - kLeft + jr0;
    live = 0;
#pragma unroll
    for (int s = 0; s < kSteps; ++s)
      if (jr0 + kJStep * s < kPooled && jt + kJStep * s >= 0 && jt + kJStep * s < Wp) live |= 1u << s;
    v_img = static_cast<long>(img) * Hp;
    m_img = static_cast<long>(img % p.mask_n) * Hp;
  }

  // Input row y into slot `dst` once `empty` completes phase `parity`; every warp arrives on `full` once it has written its share.
  __device__ __forceinline__ void row(const TcParams& p, int y, uint8_t* dst, uint64_t* full, uint64_t* empty, uint32_t parity) const {
    const int Wp = p.W >> 1;
    const uint32_t row_live = y >= 0 && y < p.H ? live : 0u;
    const __half* const vp = p.unpool_in + ((v_img + (y >> 1)) * Wp + jt) * 64 + 8 * c;
    const uint8_t* const mp = p.unpool_mask + ((m_img + (y >> 1)) * Wp + jt) * 64 + 8 * c;
    uint4 v[kSteps];
    uint2 m[kSteps];
#pragma unroll
    for (int s = 0; s < kSteps; ++s) {
      v[s] = make_uint4(0u, 0u, 0u, 0u);
      m[s] = make_uint2(0u, 0u);
      if (row_live & (1u << s)) {
        v[s] = __ldg(reinterpret_cast<const uint4*>(vp + s * kJStep * 64));
        m[s] = __ldg(reinterpret_cast<const uint2*>(mp + s * kJStep * 64));
      }
    }
    mbar_wait(empty, parity);
#pragma unroll
    for (int dx = 0; dx < 2; ++dx) {
      const int px = px0 + dx;
      uint8_t* const d = dst + px * 128 + ((c ^ (px & 7)) << 4);
      const uint32_t code = 0x01010101u * static_cast<uint32_t>(2 * (y & 1) + dx);
#pragma unroll
      for (int s = 0; s < kSteps; ++s) {
        if (jr0 + kJStep * s >= kPooled || px + 2 * kJStep * s < 0 || px + 2 * kJStep * s >= kHalo) continue;
        const uint32_t lo = __vcmpeq4(m[s].x, code), hi = __vcmpeq4(m[s].y, code);  // 0xFF per matching byte
        const uint4 o = make_uint4(v[s].x & __byte_perm(lo, 0u, 0x1100), v[s].y & __byte_perm(lo, 0u, 0x3322),
                                   v[s].z & __byte_perm(hi, 0u, 0x1100), v[s].w & __byte_perm(hi, 0u, 0x3322));
        *reinterpret_cast<uint4*>(d + s * 2 * kJStep * 128) = o;
      }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes, read by wgmma
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(full);
  }
};

// TcCta: what k_conv_tc and k_conv_tn share -- the CTA's shared-memory carve-up (see tc_smem_bytes), its place in the
// (strip, row block, cout tile, image) grid, and warpgroup 0's producers that fill the two rings.
// UNPOOL (ROLL only): warps 0, 2 and 3 expand the halo rows from the pooled input (HaloUnpool) instead of warp 0's TMA.
template <int K, bool ROLL, int KW, bool PK2, int N, bool UNPOOL = false>
struct TcCta {
  static constexpr int RK = kRows + K - 1;           // halo rows one row block reads (per chunk)
  static constexpr int kSlots = tc_slots(K, ROLL);
  static constexpr int kPad = (K - 1) / 2, kPadW = (KW - 1) / 2;
  static constexpr int b_bytes = N * 128;
  static constexpr int b_stride = tc_b_stride(N);
  static constexpr int UPC = PK2 ? KW * RK : RK;     // halo units per (row block, chunk)
  static_assert(!UNPOOL || (ROLL && KW == K), "the unpooled input is one 64-channel chunk, not window-folded");
  static constexpr int kExpandThreads = 96;          // UNPOOL: warps 0, 2, 3
  uint8_t *a_slots, *b_stages, *stage;
  uint64_t *a_full, *a_empty, *b_full, *b_empty;   // [kSlots], [kSlots], [kBStages], [kBStages]
  int kBStages, n0, img, x0, NC, npairs, y_base, n_units;

  __device__ __forceinline__ TcCta(const TcParams& p, uint8_t* smem, int stage_bytes) {
    a_slots = smem;
    b_stages = smem + kSlots * kSlotBytes;
    kBStages = p.b_stages;
    stage = b_stages + kBStages * b_stride;
    a_full = reinterpret_cast<uint64_t*>(stage + stage_bytes);
    a_empty = a_full + kSlots;
    b_full = a_empty + kSlots;
    b_empty = b_full + kBStages;
    const int strip = blockIdx.x % p.strips, rowblk = blockIdx.x / p.strips;
    n0 = blockIdx.y * N;
    img = PK2 ? 2 * blockIdx.z : blockIdx.z;
    x0 = strip * 128;
    NC = ROLL ? 1 : p.chunks;
    const int total_pairs = (p.H + kRows - 1) / kRows;
    const int pair0 = rowblk * p.pairs_per_cta;
    npairs = min(p.pairs_per_cta, total_pairs - pair0);
    y_base = pair0 * kRows;                          // first output row of this CTA
    n_units = ROLL ? npairs * kRows + K - 1 : npairs * NC * UPC;
  }

  __device__ __forceinline__ void init_barriers() const {
    // UNPOOL: each expanding warp arrives once it has written its share of a halo row (no transaction bytes)
    for (int i = 0; i < kSlots; ++i) { mbar_init(a_full + i, UNPOOL ? kExpandThreads / 32 : 1); mbar_init(a_empty + i, kEmptyArrivals); }
    for (int i = 0; i < kBStages; ++i) { mbar_init(b_full + i, 1); mbar_init(b_empty + i, kEmptyArrivals); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }

  // Warpgroup 0: warp 0 streams the halo rows, warp 1 the weight tiles; the other producer threads have nothing to do.
  // UNPOOL: warps 0, 2 and 3 expand the halo rows.
  __device__ __forceinline__ void produce(const CUtensorMap& map_a, const CUtensorMap& map_b, const TcParams& p, int warp, int lane) const {
    // 384 threads start with 168 registers each; the producers need few, the consumers (the accumulators, the split sums,
    // the epilogue's packed outputs) many: 128 x 40 + 256 x 232 = 64 512 <= 65 536.  UNPOOL: the expanding producers keep a
    // row's loads in flight (36 registers of values and masks per thread): 128 x 88 + 256 x 208 = 64 512
    if constexpr (UNPOOL) asm volatile("setmaxnreg.dec.sync.aligned.u32 88;" ::: "memory");
    else asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (UNPOOL && warp != 1) {
      // ===== halo-row expansion =====
      HaloUnpool<K, kExpandThreads> h(threadIdx.x - (warp >= 2 ? 32 : 0));
      h.strip(p, img, x0);
      for (int u = 0; u < n_units; ++u) {
        const int slot = u % kSlots;
        h.row(p, y_base - kPad + u, a_slots + slot * kSlotBytes, a_full + slot, a_empty + slot, ((u / kSlots) & 1) ^ 1);
      }
    } else if (!UNPOOL && warp == 0 && lane == 0) {
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
  }
};

__device__ __forceinline__ uint8_t* tc_smem_base() {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
}

template <int K, bool ROLL, int KW, bool PK2, int N, bool SPLIT>
__global__ void __launch_bounds__(kTcThreads, 1)
k_conv_tc(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const __grid_constant__ TcParams p,
          const __grid_constant__ TcConsts cst) {
  static_assert(!PK2 || (!ROLL && KW == K), "image-pair tiles use the chunked kernel");
  static_assert(!SPLIT || (!ROLL && N <= 64), "split mode: chunked kernel, segment sums in registers");
  using Cta = TcCta<K, ROLL, KW, PK2, N>;
  static_assert(tc_stages(K, ROLL, N, 0) > 0, "halo ring + 3 weight stages must fit in shared memory");
  constexpr int RK = Cta::RK, kSlots = Cta::kSlots, b_stride = Cta::b_stride;
  constexpr int F = N / 2;                           // accumulator registers per thread per output row
  const Cta cta(p, tc_smem_base(), 0);
  const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) cta.init_barriers();
  __syncthreads();
  if (wg == 0) {
    cta.produce(map_a, map_b, p, warp, lane);
    return;
  }
  const int kBStages = cta.kBStages, n0 = cta.n0, img = cta.img, x0 = cta.x0, NC = cta.NC, npairs = cta.npairs;
  const int y_base = cta.y_base, n_units = cta.n_units;
  uint64_t *const a_full = cta.a_full, *const a_empty = cta.a_empty, *const b_full = cta.b_full, *const b_empty = cta.b_empty;

  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
  // ===== consumers: warpgroup g = wg - 1 owns tile rows (pixels) [64 g, 64 g + 64) =====
  const int g = wg - 1;
  const int m0 = 16 * (warp & 3) + (lane >> 2);    // this thread's accumulator rows: m0 and m0 + 8
  const int img_c = PK2 ? img + g : img;
  const int x_m0 = (PK2 ? 0 : x0 + 64 * g) + m0;
  // PK2: the second image's 64-pixel box sits 64 rows into the slot; otherwise pixel 64 g of the halo row is 64 g rows in
  const uint32_t a_base = smem_u32(cta.a_slots) + static_cast<uint32_t>(g * 64 * 128), b_base = smem_u32(cta.b_stages);
  const bool releaser = lane == 0;
  const int q = lane & 3;
  // N = 64 store / dropout / unpool epilogues are deferred: block j's outputs are staged in registers, and their stores go
  // out one slice per tap row of block j + 1, right after that tap row's first MMA group is committed, so they drain while
  // the tensor core works (the last block's are flushed at the end).  The walk is instantiated once per epilogue kind so
  // that the staged registers are not live next to the immediate pool epilogue, which would then spill.
  constexpr bool kDefer = N == 64 && !SPLIT;
  auto walk = [&](auto defer_tag) {
    constexpr bool D = decltype(defer_tag)::value;
    float acc[kRows][F];
    float accr[SPLIT ? kRows : 1][SPLIT ? F : 1];
    EpiStage<D ? N : 32> ep;
    bool pending = false;
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
            if constexpr (D) {
              if (kw == 0 && rep == 0 && ch == 0 && kwo == 0 && pending) {
                // the previous block's chunks i with i K / 8 == kh: every chunk goes out during the first chunk's K tap rows
#pragma unroll
                for (int i = 0; i < EpiStage<N>::kChunks; ++i)
                  if ((i * K) / EpiStage<N>::kChunks == kh) epilogue_flush<N>(p, ep, i, x_m0, n0, q);
              }
            }
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
      if constexpr (D) {
        epilogue_stage<N>(p, cst, acc, img_c, y0, x_m0, n0, q, ep);
        pending = true;
      } else {
        epilogue_block<N>(p, cst, acc, img_c, y0, x_m0, n0, lane);
      }
    }
    if constexpr (D) {
      if (pending) {
#pragma unroll
        for (int i = 0; i < EpiStage<N>::kChunks; ++i) epilogue_flush<N>(p, ep, i, x_m0, n0, q);
      }
    }
  };
  if constexpr (kDefer) {
    if (!p.pool_out && !p.out_f32) walk(std::true_type{});
    else walk(std::false_type{});
  } else {
    walk(std::false_type{});
  }
}

// k_conv_tn: the Cin = 64 -> 64-wide half convolutions of k_conv_tc<K, true, KW, false, 64> with the GEMM transposed
// (run for K = 7, see tc_choose_kernel).
// There, each consumer's m64n64k16 reads a 2 KB pixel tile and a 2 KB weight tile for 64 K multiply-adds: 0.0625 B of
// shared-memory operand reads per MAC.  Here D^T[64 cout x 128 px] = W[64 cout x 16 cin] * X^T[16 cin x 128 px] is ONE
// m64n128k16 per (output row, tap, K step): 2 KB of weights + 4 KB of pixels, 0.047 B per MAC.  No layout changes: the
// weight stage [cout][cin] is a K-major A tile as it is, and a halo row [px][64 cin] a K-major B tile with N = 128 pixels,
// shifted by kw pixels through its start address (the swizzle phase follows the absolute address, see make_desc).
//  * Producers, rings and row-block walk: TcCta<K, true, KW, false, 64>, as k_conv_tc.
//  * Consumer g computes output row y0 + g of every block: 128 pixels x 64 couts, 64 fp32 accumulators per thread
//    (d[4 j + 2 h + e] = cout 16 warp + lane / 4 + 8 h, pixel 8 j + 2 (lane % 4) + e).  Per output element the adds run in
//    k_conv_tc's order -- tap row, tap column, K step, onto a zeroed accumulator -- so the results are the same bits.
//  * Epilogue through shared memory: bias / BN / ReLU -> half, then stmatrix .trans into a [2 rows][128 px][64 ch] staging
//    tile in SWIZZLE_128B chunk order (one 16-byte chunk = 8 channels of a pixel).  Once both rows are there (named barrier
//    over the two consumers) the stores go out in 16-byte units (pixel, 8 channels), one slice per tap row of the next
//    block right after its first MMA group is committed, the last block's at the end: a store, dropout (keep bits drawn
//    once per pixel) and a store, or 2x2 max-pool + argmax over four staged pixels.  A second barrier before the next
//    staging keeps the single tile safe.  There is no max-unpool scatter: a max-unpool that follows is expanded by its
//    consumer as it loads (UNPOOL below) or runs as its own kernel.
//  * UNPOOL: the input is a max-unpool (Basic's upsample4 .. upsample2 -> conv_decode4 .. conv_decode2); warps 0, 2 and 3
//    expand each halo row from the pooled tensor and its mask (HaloUnpool) instead of warp 0's TMA, so the unpooled
//    tensor, three quarters zeros, is neither written nor read back.  The consumers are unchanged.
constexpr int kTnStageBytes = kRows * 128 * 128;  // [kRows][128 px][64 ch] half
constexpr int kTnUnits = kRows * 128 * 8 / 256;   // 16-byte store units per consumer thread per block (2x2 pool: 2)

__device__ __forceinline__ void stmatrix_x4_trans(uint32_t addr, const uint32_t (&r)[4]) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r[0]), "r"(r[1]), "r"(r[2]),
               "r"(r[3])
               : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }  // warpgroups 1 and 2
// staged chunk c (channels 8 c .. 8 c + 7 of the tile) of pixel px, output row r of the block
__device__ __forceinline__ uint32_t tn_chunk(uint32_t s_base, int r, int px, int c) {
  return s_base + static_cast<uint32_t>(r * (128 * 128) + px * 128 + ((c ^ (px & 7)) << 4));
}
template <int K, int KW, bool UNPOOL = false>
__global__ void __launch_bounds__(kTcThreads, 1)
k_conv_tn(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const __grid_constant__ TcParams p,
          const __grid_constant__ TcConsts cst) {
  using Cta = TcCta<K, true, KW, false, 64, UNPOOL>;
  constexpr int kSlots = Cta::kSlots, b_stride = Cta::b_stride;
  static_assert(K >= kRows, "a block's own halo rows are released by its tap rows kh < kRows");
  static_assert(tc_stages(K, true, 64, kTnStageBytes) > 0, "halo ring + staging tile + 3 weight stages must fit in shared memory");
  const Cta cta(p, tc_smem_base(), kTnStageBytes);
  const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) cta.init_barriers();
  __syncthreads();
  if (wg == 0) {
    cta.produce(map_a, map_b, p, warp, lane);
    return;
  }
  if constexpr (UNPOOL) asm volatile("setmaxnreg.inc.sync.aligned.u32 208;" ::: "memory");
  else asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
  const int g = wg - 1;             // output row y0 + g of every block
  const int t = threadIdx.x - 128;  // consumer thread
  const int n0 = cta.n0, img = cta.img, x0 = cta.x0, kBStages = cta.kBStages;
  const uint32_t a_base = smem_u32(cta.a_slots), b_base = smem_u32(cta.b_stages), s_base = smem_u32(cta.stage);
  const bool releaser = lane == 0;
  const int c_lo = n0 + 16 * (warp & 3) + (lane >> 2);  // this thread's couts (rows of D^T): c_lo, c_lo + 8

  // The staged block's first row.  Store unit i of this thread is chunk t % 8 of pixel t / 8 + 32 (i % 4) of row i / 4
  // (pool: pooled pixel t / 8 + 32 i).  Lane l draws the dropout keep bits of the pixel of unit l / 4 of lane 8 (l % 4)
  // (two words: the tile's 64 channels) and shuffles them to its owners.
  int ys = 0;
  bool pending = false;
  uint32_t keep[2] = {0xFFFFFFFFu, 0xFFFFFFFFu};
  const int c = t & 7;
  auto flush_store = [&](int i) {
    const int px = (t >> 3) + 32 * (i & 3), y = ys + (i >> 2), x = x0 + px;
    uint4 v = lds128(tn_chunk(s_base, i >> 2, px, c));
    if (p.has_drop) {
      const int src = 4 * i + (lane >> 3);
      const uint32_t k0 = __shfl_sync(0xffffffffu, keep[0], src), k1 = __shfl_sync(0xffffffffu, keep[1], src);
      const uint32_t kb = ((c >> 2) ? k1 : k0) >> (8 * (c & 3));  // the keep bits of the chunk's 8 channels
      v = make_uint4(drop_word(v.x, kb, 0, p.drop_scale), drop_word(v.y, kb, 2, p.drop_scale), drop_word(v.z, kb, 4, p.drop_scale),
                     drop_word(v.w, kb, 6, p.drop_scale));
    }
    if (y < p.H && x < p.W)
      *reinterpret_cast<uint4*>(static_cast<__half*>(p.out) + ((static_cast<size_t>(img) * p.H + y) * p.W + x) * p.cout_total + n0 + 8 * c) = v;
  };
  auto flush_pool = [&](int i) {  // the window's four staged pixels, in scan order
    const int pp = (t >> 3) + 32 * i, x = x0 + 2 * pp;
    const uint4 a = lds128(tn_chunk(s_base, 0, 2 * pp, c)), b = lds128(tn_chunk(s_base, 0, 2 * pp + 1, c));
    const uint4 cc = lds128(tn_chunk(s_base, 1, 2 * pp, c)), d = lds128(tn_chunk(s_base, 1, 2 * pp + 1, c));
    const uint32_t av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w}, cv[4] = {cc.x, cc.y, cc.z, cc.w}, dv[4] = {d.x, d.y, d.z, d.w};
    uint32_t best[4], arg[4];
#pragma unroll
    for (int w = 0; w < 4; ++w) best[w] = pool2x2(av[w], bv[w], cv[w], dv[w], arg[w]);
    if (ys + 1 < p.H && x + 1 < p.W) {
      const size_t o = ((static_cast<size_t>(img) * (p.H >> 1) + (ys >> 1)) * (p.W >> 1) + (x >> 1)) * p.cout_total + n0 + 8 * c;
      *reinterpret_cast<uint4*>(p.pool_out + o) = make_uint4(best[0], best[1], best[2], best[3]);
      *reinterpret_cast<uint2*>(p.pool_mask + o) = make_uint2(arg[0] | (arg[1] << 16), arg[2] | (arg[3] << 16));
    }
  };
  // the staged block's units that go out during tap row kh: every unit during the K tap rows
  auto flush_slice = [&](int kh) {
    if (p.has_drop && kh == 0) {
      const int i = lane >> 2, px = (t >> 5) * 4 + (lane & 3) + 32 * (i & 3), y = ys + (i >> 2), x = x0 + px;
      uint32_t bits[4];
      dropout_bits128_nl(p.seed, *p.frame, p.drop_nl + img, static_cast<uint32_t>(y * p.W + x), n0 >> 7, bits);
      keep[0] = (n0 & 64) ? bits[2] : bits[0];
      keep[1] = (n0 & 64) ? bits[3] : bits[1];
    }
#pragma unroll
    for (int i = 0; i < kTnUnits; ++i) {
      if (p.pool_out) {
        if (i < 2 && (i * K) / 2 == kh) flush_pool(i);
      } else if ((i * K) / kTnUnits == kh) {
        flush_store(i);
      }
    }
  };

  float acc[64];
  int st = 0;
  uint32_t b_phase = 0;
  int waited = 0;  // halo units whose TMA has been observed
  for (int j = 0; j < cta.npairs; ++j) {
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    const int base_u = j * kRows;
    for (int kh = 0; kh < K; ++kh) {
      while (waited <= base_u + kh + kRows - 1 && waited < cta.n_units) {
        mbar_wait(cta.a_full + waited % kSlots, (waited / kSlots) & 1);
        ++waited;
      }
      const uint32_t x_row = a_base + ((base_u + g + kh) % kSlots) * kSlotBytes;
      int prev_st = -1;
#pragma unroll
      for (int kw = 0; kw < KW; ++kw) {
        mbar_wait(cta.b_full + st, b_phase);
        const uint32_t w_addr = b_base + st * b_stride;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma(acc, make_desc(w_addr + 32 * k), make_desc(x_row + kw * 128 + 32 * k));
        wgmma_commit();
        if (kw == 0 && pending) flush_slice(kh);
        // keep one group in flight: the previous one has retired, so its weight stage goes back to the producer
        wgmma_wait<1>();
        if (prev_st >= 0 && releaser) mbar_arrive(cta.b_empty + prev_st);
        prev_st = st;
        if (++st == kBStages) { st = 0; b_phase ^= 1; }
      }
      wgmma_wait<0>();
      fence_acc(acc);
      if (releaser) {
        mbar_arrive(cta.b_empty + prev_st);
        // k_conv_tc's release rule holds: consumer 1 reads halo row base_u + kh at tap row kh - 1, consumer 0 at tap row kh --
        // one tap row earlier, never later -- so once both have passed tap row kh neither reads it again in this block, and
        // rows >= kRows are the next block's (released by its tap rows)
        if (kh < kRows) mbar_arrive(cta.a_empty + (base_u + kh) % kSlots);
      }
    }
    consumers_sync();  // both consumers have flushed the previous block out of the staging tile
    {
      // lane l addresses row l % 8 of matrix l / 8 = (h, j) = (l / 8 % 2, 2 jp + l / 16): pixel 8 j + l % 8, chunk 2 warp + h
      const int rr = lane & 7, h = (lane >> 3) & 1;
      const uint32_t addr = s_base + static_cast<uint32_t>(g * (128 * 128) + (8 * (lane >> 4) + rr) * 128 + (((2 * (warp & 3) + h) ^ rr) << 4));
#pragma unroll
      for (int jp = 0; jp < 8; ++jp) {
        uint32_t r4[4];
#pragma unroll
        for (int m = 0; m < 4; ++m) {
          const int mh = m & 1, mj = 2 * jp + (m >> 1);
          const __half2 hv = __floats2half2_rn(affine(p, cst, acc[4 * mj + 2 * mh], c_lo + 8 * mh),
                                               affine(p, cst, acc[4 * mj + 2 * mh + 1], c_lo + 8 * mh));
          r4[m] = *reinterpret_cast<const uint32_t*>(&hv);
        }
        stmatrix_x4_trans(addr + jp * 16 * 128, r4);
      }
    }
    consumers_sync();  // both rows staged
    ys = cta.y_base + j * kRows;
    pending = true;
  }
  if (pending)
    for (int kh = 0; kh < K; ++kh) flush_slice(kh);
}

// k_conv_stack's shared memory: the resident weights (per kw the tap rows kh = 0 .. K-1, 0 .. K-2 of [16 cout][64 cin] half:
// 2 K - 1 blocks of 2 KB), then as many halo-row slots as fit, then the mbarriers.
__host__ __device__ constexpr int stack_w_bytes(int K) { return K * (2 * K - 1) * 16 * 128; }
__host__ __device__ constexpr int stack_slots(int K) { return (227 * 1024 - 1024 - 256 - stack_w_bytes(K)) / kSlotBytes; }
__host__ __device__ constexpr int stack_smem_bytes(int K) {
  return 1024 + stack_w_bytes(K) + stack_slots(K) * kSlotBytes + (2 * stack_slots(K) + 2) * 8;
}

// Epilogue of one output row of k_conv_stack for one consumer thread: pixels m0 and m0 + 8 (h = 0, 1), channels 8 j + 2 q + e.
__device__ __forceinline__ void epilogue_row16(const TcParams& p, const TcConsts& cst, const float (&a)[8], int img, int y, int x_m0, int q) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int x = x_m0 + 8 * h;
    const size_t pix = (static_cast<size_t>(img) * p.H + y) * p.W + x;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int c = 8 * j + 2 * q;
      const float2 v = make_float2(affine(p, cst, a[4 * j + 2 * h], c), affine(p, cst, a[4 * j + 2 * h + 1], c + 1));
      if (x < p.W) *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.out) + pix * p.cout_total + c) = v;
    }
  }
}

// One input row of k_conv_stack at phase PH: its MMAs, then output row r - (K - 1) (slot K-1-PH) moved out to `v` and its
// slot zeroed.  The epilogue runs on `v` outside the phase switch, once.
template <int K, int PH>
__device__ __forceinline__ void stack_row(float (&acc)[K][8], uint32_t a_row, uint32_t w_base, float (&v)[8]) {
  if constexpr (PH < K) {
    constexpr int kKwBytes = (2 * K - 1) * 16 * 128;  // the resident rows of one tap column
    wgmma_fence();
#pragma unroll
    for (int kw = 0; kw < K; ++kw)
#pragma unroll
      for (int k = 0; k < 4; ++k)  // B = tap rows PH .. PH + K - 1 (mod K) of tap column kw
        wgmma_stack(acc, make_desc(a_row + kw * 128 + 32 * k), make_desc(w_base + kw * kKwBytes + PH * 16 * 128 + 32 * k));
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc(acc);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      v[i] = acc[K - 1 - PH][i];
      acc[K - 1 - PH][i] = 0.f;
    }
  }
}

// The halo producer of k_conv_stack<K, true>, run by all four warps of warpgroup 0 (HaloUnpool): per run of output rows
// within one strip, input rows y_start - pad .. y_end - 1 + pad.
template <int K>
__device__ __forceinline__ void stack_unpool_producer(const TcParams& p, uint8_t* a_slots, uint64_t* a_full, uint64_t* a_empty,
                                                      long t_begin, long t_end) {
  constexpr int kPad = (K - 1) / 2;
  constexpr int kSlots = stack_slots(K);
  HaloUnpool<K, 128> h(threadIdx.x);
  uint32_t u = 0;
  for (long t = t_begin; t < t_end;) {
    const int col = static_cast<int>(t / p.H), y_start = static_cast<int>(t % p.H);
    const int n_out = static_cast<int>(min(static_cast<long>(p.H - y_start), t_end - t));
    h.strip(p, col / p.strips, (col % p.strips) * 128);
    for (int r = 0; r < n_out + K - 1; ++r, ++u) {
      const int slot = u % kSlots;
      h.row(p, y_start - kPad + r, a_slots + slot * kSlotBytes, a_full + slot, a_empty + slot, ((u / kSlots) & 1) ^ 1);
    }
    t += n_out;
  }
}

// Cin = 64 -> 16 float channels, K x K (K = 3, 7): the float-logits layers (the composed classifier, Standard's conv1_1_D).
// An m64n16k16 MMA reads a 2 KB A tile for 16 output columns, which makes the 16-wide k_conv_tc tile bound by shared-memory
// operand reads.  Here the K tap rows are stacked along N instead: ONE m64n{16K}k16 per (kw, K step) of input row i computes
// the contributions of all K tap rows of tap column kw, tap row kh to output row i + pad - kh.  A operand reads drop K-fold
// and the layer is bound by the tensor rate.
//  * Output rows live in a ring of K accumulator slots of 8 fp32 per thread (64 pixels x 16 channels), counted downwards:
//    relative output row y (from the run's first row) sits in slot (-y) mod K, so at phase ph = r mod K of relative input row
//    r, slot j takes tap row (ph + j) mod K.  The slots keep fixed registers and the weights rotate instead: per tap column
//    the rows kh = 0 .. K-1, 0 .. K-2 are resident, and phase ph's B operand is the K-row window starting at row ph.  The
//    phase selects one of K copies of the issue code.  After input row r, output row r - (K - 1) (slot K-1-ph) is complete:
//    it is stored and its slot zeroed for the row that enters next.  Per output pixel the adds run in the order of k_conv_tc
//    -- tap row kh ascending, then kw, then the 4 K steps -- onto a zeroed accumulator, out-of-image rows included
//    (zero-filled by TMA), so the results are the same bits.
//  * The weights (182 KB for K = 7, 30 KB for K = 3) are loaded once per CTA: per kw one TMA box {64 cin, 16 cout, 1, K kh}
//    out of the [kh][kw][cout][cin] tensor, which lands [kh][16][64]; the weight warp copies rows 0 .. K-2 behind it.  What
//    is left of shared memory holds the halo ring (2 slots for K = 7, 11 for K = 3).
//  * A CTA emits rows [b R, b R + R) of the flattened (image, strip, row) range; each maximal run of rows within one strip
//    first walks K - 1 warm-up input rows, whose MMAs only feed rows that are not emitted.  Every input row is read by one
//    step and then released, so the halo ring is pure prefetch.
//  * UNPOOL: the input is a max-unpool (Basic's upsample1 -> conv_decode1); the four producer warps expand each halo row
//    from the pooled tensor and its mask (stack_unpool_producer) instead of one TMA box, so the unpooled tensor, three
//    quarters zeros, is neither written nor read back.  The consumers are unchanged.
template <int K, bool UNPOOL = false>
__global__ void __launch_bounds__(kTcThreads, 1)
k_conv_stack(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const __grid_constant__ TcParams p,
             const __grid_constant__ TcConsts cst) {
  constexpr int kPad = (K - 1) / 2;
  constexpr int kSlots = stack_slots(K);
  constexpr int kBlock = 16 * 128;                  // one tap row: [16 cout][64 cin] half
  constexpr int kKwBytes = (2 * K - 1) * kBlock;    // one tap column
  static_assert(stack_smem_bytes(K) <= 227 * 1024 && kSlots >= 2 && K <= 7, "weights + halo ring must fit in shared memory");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* w_smem = smem;
  uint8_t* a_slots = smem + stack_w_bytes(K);
  uint64_t* a_full = reinterpret_cast<uint64_t*>(a_slots + kSlots * kSlotBytes);  // [kSlots]
  uint64_t* a_empty = a_full + kSlots;                                             // [kSlots]
  uint64_t* w_full = a_empty + kSlots;   // TMA landed tap rows 0 .. K-1 of every column
  uint64_t* w_ready = w_full + 1;        // ... and the copies of rows 0 .. K-2 behind them

  const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long rows = static_cast<long>(p.N_batch) * p.strips * p.H;
  const long t_begin = static_cast<long>(blockIdx.x) * p.rows_per_cta;
  const long t_end = min(t_begin + p.rows_per_cta, rows);

  if (threadIdx.x == 0) {
    // UNPOOL: each of the four producer warps arrives once it has written its share of a halo row
    for (int i = 0; i < kSlots; ++i) { mbar_init(a_full + i, UNPOOL ? 4 : 1); mbar_init(a_empty + i, kEmptyArrivals); }
    mbar_init(w_full, 1);
    mbar_init(w_ready, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  if (wg == 0) {
    // UNPOOL: the expanding producers keep a row's loads in flight (30 registers of values and masks per thread):
    // 128 x 80 + 256 x 208 = 63 488 <= 64 512
    if constexpr (UNPOOL) asm volatile("setmaxnreg.dec.sync.aligned.u32 80;" ::: "memory");
    else asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp == 0 && lane == 0 && !UNPOOL) {
      // ===== halo-row producer: per run, input rows y_start - pad .. y_end - 1 + pad =====
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_a)) : "memory");
      uint32_t u = 0;
      for (long t = t_begin; t < t_end;) {
        const int col = static_cast<int>(t / p.H), y_start = static_cast<int>(t % p.H);
        const int n_out = static_cast<int>(min(static_cast<long>(p.H - y_start), t_end - t));
        const int img = col / p.strips, x0 = (col % p.strips) * 128;
        for (int r = 0; r < n_out + K - 1; ++r, ++u) {
          const int slot = u % kSlots;
          mbar_wait(a_empty + slot, ((u / kSlots) & 1) ^ 1);
          mbar_expect_tx(a_full + slot, static_cast<uint32_t>((128 + K - 1) * 128));
          tma_load_4d(a_slots + slot * kSlotBytes, &map_a, a_full + slot, 0, x0 - kPad, y_start - kPad + r, img);
        }
        t += n_out;
      }
    } else if (warp == 1) {
      // ===== weights, once: TMA lands rows 0 .. K-1 of each tap column, the warp copies rows 0 .. K-2 behind them (whole
      // 1 KB swizzle groups, so the SWIZZLE_128B phase is the same at the copy), and every window of K consecutive rows
      // is the B operand of one phase =====
      if (lane == 0) {
        mbar_expect_tx(w_full, static_cast<uint32_t>(K * K * kBlock));
        for (int kw = 0; kw < K; ++kw) tma_load_4d(w_smem + kw * kKwBytes, &map_b, w_full, 0, 0, kw, 0);
      }
      mbar_wait(w_full, 0);
      for (int kw = 0; kw < K; ++kw) {
        const uint4* src = reinterpret_cast<const uint4*>(w_smem + kw * kKwBytes);
        uint4* dst = reinterpret_cast<uint4*>(w_smem + kw * kKwBytes + K * kBlock);
        for (int i = lane; i < (K - 1) * kBlock / 16; i += 32) dst[i] = src[i];
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes, read by wgmma
      __syncwarp();
      if (lane == 0) mbar_arrive(w_ready);
    }
    if constexpr (UNPOOL) stack_unpool_producer<K>(p, a_slots, a_full, a_empty, t_begin, t_end);
    return;
  }

  if constexpr (UNPOOL) asm volatile("setmaxnreg.inc.sync.aligned.u32 208;" ::: "memory");
  else asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
  // ===== consumers: warpgroup g = wg - 1 owns pixels [64 g, 64 g + 64) of the strip =====
  const int g = wg - 1;
  const int m0 = 16 * (warp & 3) + (lane >> 2);
  const uint32_t a_base = smem_u32(a_slots) + static_cast<uint32_t>(g * 64 * 128), w_base = smem_u32(w_smem);
  const bool releaser = lane == 0;
  mbar_wait(w_ready, 0);
  float acc[K][8];
  uint32_t u = 0;
  for (long t = t_begin; t < t_end;) {
    const int col = static_cast<int>(t / p.H), y_start = static_cast<int>(t % p.H);
    const int n_out = static_cast<int>(min(static_cast<long>(p.H - y_start), t_end - t));
    const int img = col / p.strips, x_m0 = (col % p.strips) * 128 + 64 * g + m0;
    const int n_in = n_out + K - 1;
#pragma unroll
    for (int s = 0; s < K; ++s)
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[s][i] = 0.f;
    for (int r = 0; r < n_in; ++r) {  // input row y_start - pad + r: its tap row kh feeds relative output row r - kh
      const int slot = u % kSlots;
      mbar_wait(a_full + slot, (u / kSlots) & 1);
      const uint32_t a_row = a_base + slot * kSlotBytes;
      float v[8];
      switch (r % K) {
        case 0: stack_row<K, 0>(acc, a_row, w_base, v); break;
        case 1: stack_row<K, 1>(acc, a_row, w_base, v); break;
        case 2: stack_row<K, 2>(acc, a_row, w_base, v); break;
        case 3: stack_row<K, 3>(acc, a_row, w_base, v); break;
        case 4: stack_row<K, 4>(acc, a_row, w_base, v); break;
        case 5: stack_row<K, 5>(acc, a_row, w_base, v); break;
        default: stack_row<K, 6>(acc, a_row, w_base, v); break;
      }
      if (releaser) mbar_arrive(a_empty + slot);
      ++u;
      // output row y_start + r - (K - 1) got its last tap row (rows before y_start are warm-up, not emitted)
      if (r >= K - 1) epilogue_row16(p, cst, v, img, y_start + r - (K - 1), x_m0, lane & 3);
    }
    t += n_out;
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

// every convolution kernel's signature
using TcKernel = void (*)(CUtensorMap, CUtensorMap, TcParams, TcConsts);

}  // namespace

struct ConvTcPlan {
  CUtensorMap map_a, map_b;
  TcParams p;
  TcConsts cst;
  dim3 grid;
  size_t smem;
  int k;
  int kw;             // filter width the kernel walks (== k, or 1 for a window-folded layer)
  TcKernel kern = nullptr;  // set by tc_choose_kernel
  double rows_ratio = 1.0;  // k_conv_stack: input rows it runs the MMAs of / output rows (the warm-up rows of every run)
  DevBuf w_own;       // weights the plan owns (the composed classifier)
};

namespace {
// one 64-channel input chunk: the halo rows persist in the ring while a CTA walks down its strip (ROLL)
bool tc_roll(const TcParams& p) { return p.chunks == 1 && !p.split; }
// k_conv_stack: the 64 -> 16 float-logits layers, K = 3 / 7
bool tc_stacked(const ConvTcPlan& plan) { return tc_roll(plan.p) && plan.p.n_tile == 16 && plan.k > 1; }
// two images per 128-pixel M tile (PK2): chunked 3x3 layers at most 64 pixels wide
// k_conv_tn: every Cin = 64, K = 7 layer with 64-wide half output tiles.  The K = 3 layers stay on k_conv_tc: on
// k_conv_tn Standard's conv1_2_D (352 x 1024, T = 12) took 0.75 ms in one session and 1.77 ms in another, against
// k_conv_tc's steady 1.35 ms (H100 80GB HBM3, 700 W).
bool tc_tn(const ConvTcPlan& plan) { return tc_roll(plan.p) && plan.p.n_tile == 64 && plan.k == 7 && !plan.p.out_f32; }
bool tc_pk2(const ConvTcPlan& plan) {
  const TcParams& p = plan.p;
  return !tc_roll(p) && !p.split && plan.k == 3 && p.W <= 64 && p.N_batch >= 2 && p.n_tile != 16;
}

// The one place that names every instantiation: picks the kernel for the plan's shape and epilogue state, sizes its
// shared memory (and weight ring) to match and raises the kernel's dynamic shared-memory limit.  Called again whenever
// a fusion changes that state.
void tc_choose_kernel(ConvTcPlan& plan) {
  TcParams& p = plan.p;
  const int K = plan.k, n = p.n_tile;
  const bool roll = tc_roll(p), tn = tc_tn(plan);
  // per (K, ROLL, KW, PK2): the three tile widths
  auto by_n = [n](TcKernel k16, TcKernel k64, TcKernel k128) { return n == 16 ? k16 : n == 64 ? k64 : k128; };
  if (tc_stacked(plan)) {
    plan.kern = K == 3 ? k_conv_stack<3> : p.unpool_in ? k_conv_stack<7, true> : k_conv_stack<7>;
    plan.smem = stack_smem_bytes(K);
  } else {
    if (p.split) {
      if (n == 16) plan.kern = K == 7 ? k_conv_tc<7, false, 7, false, 16, true> : K == 3 ? k_conv_tc<3, false, 3, false, 16, true> : k_conv_tc<1, false, 1, false, 16, true>;
      else plan.kern = K == 7 ? k_conv_tc<7, false, 7, false, 64, true> : K == 3 ? k_conv_tc<3, false, 3, false, 64, true> : k_conv_tc<1, false, 1, false, 64, true>;
    } else if (tn) {  // KW = 1: window-folded first layer
      plan.kern = plan.kw == 1 ? k_conv_tn<7, 1> : p.unpool_in ? k_conv_tn<7, 7, true> : k_conv_tn<7, 7>;
    } else if (plan.kw == 1 && K == 3) {  // window-folded 3x3 first layer (3 x 1), 64-wide tiles
      plan.kern = k_conv_tc<3, true, 1, false, 64, false>;
    } else if (tc_pk2(plan)) {
      plan.kern = n == 64 ? k_conv_tc<3, false, 3, true, 64, false> : k_conv_tc<3, false, 3, true, 128, false>;
    } else if (roll) {
      if (K == 7) plan.kern = k_conv_tc<7, true, 7, false, 128, false>;  // 64-wide K = 7 tiles run on k_conv_tn
      else if (K == 3) plan.kern = n == 64 ? k_conv_tc<3, true, 3, false, 64, false> : k_conv_tc<3, true, 3, false, 128, false>;
      else plan.kern = by_n(k_conv_tc<1, true, 1, false, 16, false>, k_conv_tc<1, true, 1, false, 64, false>, k_conv_tc<1, true, 1, false, 128, false>);
    } else {
      if (K == 7) plan.kern = by_n(k_conv_tc<7, false, 7, false, 16, false>, k_conv_tc<7, false, 7, false, 64, false>, k_conv_tc<7, false, 7, false, 128, false>);
      else if (K == 3) plan.kern = by_n(k_conv_tc<3, false, 3, false, 16, false>, k_conv_tc<3, false, 3, false, 64, false>, k_conv_tc<3, false, 3, false, 128, false>);
      else plan.kern = by_n(k_conv_tc<1, false, 1, false, 16, false>, k_conv_tc<1, false, 1, false, 64, false>, k_conv_tc<1, false, 1, false, 128, false>);
    }
    // every kernel above fits at least 3 weight stages (static_assert in k_conv_tc / k_conv_tn)
    const int stage_bytes = tn ? kTnStageBytes : 0;
    p.b_stages = tc_stages(K, roll, n, stage_bytes);
    plan.smem = tc_smem_bytes(K, roll, n, p.b_stages, stage_bytes);
  }
  // the limit is per kernel function, not per launch: always raise it to the full 227 KB so that plans of different
  // sizes that share an instantiation cannot lower it for each other
  SIVO_CUDA(cudaFuncSetAttribute(plan.kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
}

int num_sms() {
  int dev = 0, n = 0;
  SIVO_CUDA(cudaGetDevice(&dev));
  SIVO_CUDA(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
  return std::max(1, n);
}
// Upper bound on the row blocks one CTA walks.  Long-lived CTAs amortise the prologue best, but while they run no SM
// frees up, so the extractors' short dependent kernels -- highest stream priority notwithstanding -- each wait for a
// whole CTA lifetime; this cap trades the two (unit: 2-row blocks).
constexpr int kTcMaxPpc = 48;
int tc_pick_n(const Op& op, const TensorView& out) {
  if (out.dt == DType::F32 && out.cs <= 16) return 16;  // the float logits layer
  if (op.split || op.fold_kw) return 64;                // split: the segment sums must fit in registers next to the accumulators
  return (op.cout_p % 128 == 0) ? 128 : 64;
}
// row blocks per CTA: minimise (waves over the SMs) x (blocks per CTA + ~1 block of prologue / halo overhead)
int tc_blocks_per_cta(long columns, int total_pairs, double overhead) {
  const int sms = num_sms();
  int ppc = 1;
  double best_cost = 1e30;
  for (int c = 1; c <= std::min(total_pairs, kTcMaxPpc); ++c) {
    const long ctas = columns * ceil_div(total_pairs, c);
    const double cost = static_cast<double>((ctas + sms - 1) / sms) * (c + overhead);
    if (cost < best_cost - 1e-9) { best_cost = cost; ppc = c; }
  }
  return ppc;
}
// Output rows per k_conv_stack CTA at most: bounds how long the extractors' dependent kernels wait for an SM (see kTcMaxPpc).
// Basic T=6 at 352 x 1024 (6 x 8 x 352 = 16 896 rows) is then one wave of 128-row CTAs on 132 SMs.
constexpr int kStackMaxRows = 128;
// Points a K = 3 / 7, 64 -> 16 float-logits plan at k_conv_stack.  `w` = [kh][kw][cout_rows][64] half, couts 0..15 used.
void plan_stack(ConvTcPlan& plan, void* w, int cout_rows) {
  const int K = plan.k;
  cuuint64_t dims[4] = {64, static_cast<cuuint64_t>(cout_rows), static_cast<cuuint64_t>(K), static_cast<cuuint64_t>(K)};
  cuuint64_t strides[3] = {128, static_cast<cuuint64_t>(cout_rows) * 128, static_cast<cuuint64_t>(K) * cout_rows * 128};
  cuuint32_t box[4] = {64, 16, 1, static_cast<cuuint32_t>(K)};  // one tap column: [kh][16][64]
  encode(&plan.map_b, w, 4, dims, strides, box);
  TcParams& p = plan.p;
  p.n_tile = 16;
  p.out_f32 = 1;
  // equal pieces of the flattened (image, strip, row) range, in as few waves over the SMs as kStackMaxRows allows
  const long rows = static_cast<long>(p.N_batch) * p.strips * p.H;
  const long sms = num_sms();
  const long waves = (rows + sms * kStackMaxRows - 1) / (sms * kStackMaxRows);
  p.rows_per_cta = static_cast<int>((rows + waves * sms - 1) / (waves * sms));
  const long ctas = (rows + p.rows_per_cta - 1) / p.rows_per_cta;
  long runs = 0;  // maximal runs of rows within one strip: each costs K - 1 warm-up input rows
  for (long b = 0; b < ctas; ++b) {
    const long t0 = b * p.rows_per_cta, t1 = std::min(t0 + p.rows_per_cta, rows);
    runs += (t1 - 1) / p.H - t0 / p.H + 1;
  }
  plan.rows_ratio = static_cast<double>(rows + (K - 1) * runs) / static_cast<double>(rows);
  plan.grid = dim3(static_cast<unsigned>(ctas), 1, 1);
}
}  // namespace

bool conv_tc_supported(const Op& op, const TensorView& in, const TensorView& out) {
  if (in.dt != DType::F16) return false;
  if (op.k != 1 && op.k != 3 && op.k != 7) return false;
  if (op.cout_p > kMaxCout) return false;
  if (op.fold_kw) {
    return in.cs == 8 && op.cin_p == 64 && (op.k == 3 || op.k == 7) && out.dt == DType::F16 && op.cout % 64 == 0 && out.cs == op.cout;
  }
  if (op.split) {  // `in` = the [hi Cin | lo Cin] half planes of the float input
    if (op.cin % 64 || in.cs != 2 * op.cin || out.dt != DType::F32) return false;
    return (out.cs == op.cout && op.cout % 64 == 0) || (out.cs == 16 && op.cout <= 16);
  }
  if (in.cs % 64 || op.cin != in.cs) return false;
  if (out.dt == DType::F16) return op.cout % 64 == 0 && out.cs == op.cout;
  return out.cs == 16 && op.cout <= 16;  // float logits, 16-channel pixels
}

std::shared_ptr<ConvTcPlan> conv_tc_plan(const Op& op, const TensorView& in, const TensorView& out, const void* w_tc) {
  auto plan = std::make_shared<ConvTcPlan>();
  const int K = op.k;
  const int KW = op.fold_kw ? 1 : K;
  const int n_tile = tc_pick_n(op, out);
  plan->k = K;
  plan->kw = KW;
  TcParams& p = plan->p;
  p.H = in.h; p.W = op.fold_kw ? in.w - 8 : in.w; p.N_batch = in.n;
  p.cout_total = out.cs;
  p.n_tile = n_tile;
  p.chunks = op.fold_kw ? 1 : in.cs / 64;
  p.out_f32 = out.dt == DType::F32 ? (n_tile == 16 ? 1 : 2) : 0;
  p.split = op.split ? 1 : 0;
  const bool roll = tc_roll(p), pk2 = tc_pk2(*plan);
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
    cuuint32_t box[4] = {64, static_cast<cuuint32_t>(pk2 ? 64 : 128 + K - 1), 1, 1};
    encode(&plan->map_a, in.p, 4, dims, strides, box);
  }
  {  // weights: [tap][cout_p][cin_p] half, dims (cin, cout, tap)
    const int kext = op.split ? 3 * op.cin_p : op.cin_p;  // split: [W_hi | W_lo | W_hi] per 64-channel chunk along K
    cuuint64_t dims[3] = {static_cast<cuuint64_t>(kext), static_cast<cuuint64_t>(op.cout_p), static_cast<cuuint64_t>(K * KW)};
    cuuint64_t strides[2] = {static_cast<cuuint64_t>(kext) * 2, static_cast<cuuint64_t>(op.cout_p) * kext * 2};
    cuuint32_t box[3] = {64, static_cast<cuuint32_t>(n_tile), 1};
    encode(&plan->map_b, const_cast<void*>(w_tc), 3, dims, strides, box);
  }
  p.cin_real = op.cin;
  p.acc_scale = op.split ? op.acc_scale : 1.f;
  p.seg_rows = 1;  // a segment per (chunk, tap row): 7x7 56 / 28 accumulate steps, 3x3 24 / 12, 1x1 8 / 4
  p.rz_comp = 0.216f * 1.1920929e-7f;  // x 2^-23
  p.strips = ceil_div(p.W, 128);
  const int cout_tiles = p.out_f32 == 1 ? 1 : op.cout_p / n_tile;
  const int n_z = pk2 ? ceil_div(in.n, 2) : in.n;  // PK2: an image pair per tile
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
  p.has_drop = 0; p.seed = 0; p.frame = nullptr; p.drop_nl = 0; p.drop_scale = 2.f;
  p.unpool_mask = nullptr; p.mask_n = 1; p.unpool_in = nullptr;
  p.pool_out = nullptr; p.pool_mask = nullptr;
  plan->grid = dim3(p.strips * ceil_div(total_pairs, p.pairs_per_cta), cout_tiles, n_z);
  if (tc_stacked(*plan)) plan_stack(*plan, const_cast<void*>(w_tc), op.cout_p);
  tc_choose_kernel(*plan);
  return plan;
}

void conv_tc_set_dropout(ConvTcPlan& plan, uint64_t seed, const uint64_t* frame_dev, int layer, float scale, int sample0) {
  plan.p.has_drop = 1;
  plan.p.seed = seed;
  plan.p.frame = frame_dev;
  if (sample0 < 0 || sample0 + plan.p.N_batch > (1 << 16) || layer < 0 || layer > 255)
    fail(SIVO_EINVAL, "conv_tc_set_dropout: samples [%d, %d) / layer %d outside the keep-bit counter's fields", sample0,
         sample0 + plan.p.N_batch, layer);
  plan.p.drop_nl = static_cast<uint32_t>(sample0) | (static_cast<uint32_t>(layer) << 16);
  plan.p.drop_scale = scale;
}

bool conv_tc_can_fuse_unpool(const ConvTcPlan& plan) { return !tc_tn(plan) && !plan.p.unpool_in; }

void conv_tc_set_unpool(ConvTcPlan& plan, const uint8_t* mask, int mask_n, void* out_2h_2w) {
  if (!conv_tc_can_fuse_unpool(plan)) fail(SIVO_EINVAL, "conv_tc_set_unpool: this plan's kernel has no max-unpool scatter");
  plan.p.unpool_mask = mask;
  plan.p.mask_n = mask_n;
  plan.p.out = out_2h_2w;
}

bool conv_tc_can_unpool_input(const ConvTcPlan& plan) {
  return plan.k == 7 && plan.kw == 7 && (tc_stacked(plan) || tc_tn(plan)) && !plan.p.unpool_mask;
}

void conv_tc_set_unpool_input(ConvTcPlan& plan, const void* pooled, const uint8_t* mask, int mask_n, int h, int w) {
  if (!conv_tc_can_unpool_input(plan) || 2 * h != plan.p.H || 2 * w != plan.p.W || !pooled || !mask || mask_n < 1)
    fail(SIVO_EINVAL, "conv_tc_set_unpool_input: needs a 7x7 float-logits or 64-wide half plan over the %d x %d unpooled input "
                      "(got %d x %d pooled)", plan.p.H, plan.p.W, h, w);
  plan.p.unpool_in = static_cast<const __half*>(pooled);
  plan.p.unpool_mask = mask;
  plan.p.mask_n = mask_n;
  tc_choose_kernel(plan);
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
  return !plan.p.out_f32 && !plan.p.unpool_mask && !plan.p.has_drop && (plan.p.H % 2) == 0 && (plan.p.W % 2) == 0;
}

void conv_tc_set_pool(ConvTcPlan& plan, void* pooled, uint8_t* mask) {
  plan.p.pool_out = static_cast<__half*>(pooled);
  plan.p.pool_mask = mask;
}

bool conv_tc_can_compose_classifier(const ConvTcPlan& plan) {
  return tc_tn(plan) && plan.kw == 7 && !plan.p.has_drop && !plan.p.pool_out && !plan.p.relu && !plan.p.has_bn && plan.p.cout_total == 64;
}

void conv_tc_set_composed_classifier(ConvTcPlan& plan, const Op& conv, const float* wc, const float* bc, int n_cls, float* logits) {
  const int K = 7;
  if (n_cls > 16 || conv.h_w_raw.size() != static_cast<size_t>(64) * 64 * K * K || conv.h_bias.size() < 64)
    fail(SIVO_EINVAL, "composed classifier: unexpected layer shapes");
  // W'[o][i][kh][kw] = sum_c wc[o][c] W[c][i][kh][kw] in double, rounded once to half; rows o >= n_cls stay zero.
  // Device layout [kh][kw][16][64]: the [tap][cout][cin] layout of every other weight tensor, 16 couts per tap.
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
  std::memset(&plan.cst, 0, sizeof(TcConsts));
  for (int o = 0; o < n_cls; ++o) {
    double acc = bc ? bc[o] : 0.0;
    for (int c = 0; c < 64; ++c) acc += static_cast<double>(wc[o * 64 + c]) * conv.h_bias[c];
    plan.cst.bias[o] = static_cast<float>(acc);
  }
  plan.p.cout_total = 16;
  plan.p.out = logits;
  plan_stack(plan, plan.w_own.p, 16);
  tc_choose_kernel(plan);
}

double conv_tc_rows_ratio(const ConvTcPlan& plan) { return plan.rows_ratio; }

void conv_tc_launch(const ConvTcPlan& plan, cudaStream_t s) {
  plan.kern<<<plan.grid, kTcThreads, plan.smem, s>>>(plan.map_a, plan.map_b, plan.p, plan.cst);
  SIVO_CUDA(cudaGetLastError());
}

}  // namespace sivo
