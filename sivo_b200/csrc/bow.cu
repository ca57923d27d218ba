// The bag of words on the device: TemplatedVocabulary::transform (Frame::ComputeBoW / KeyFrame::ComputeBoW) and
// ORBmatcher::SearchByBoW(KeyFrame*, Frame&) batched over keyframes.  The rules are spelled out in include/sivo_b200.h and
// oracle/bow_oracle.py.  This file is compiled with -fmad=false: every float / double intermediate is the correctly rounded result of
// the operation as written.
//
//   k_bow_descend   one warp per semantic key: per level, lanes take the node's children (CSR) and the warp keeps the smallest
//                   (distance, child position), so the first child wins ties as in the reference's strict `<`.
//   k_bow_vector    one block: the keys' words sorted in shared memory (bitonic), one BowVector entry per distinct word with the
//                   sum of its features' weights in feature order, then the normalisation's ordered sum in one thread.
//   k_sbb_sort      one block: the frame's keys sorted by (node, index), which groups each FeatureVector entry in index order.
//   k_sbb_walk      one warp per (keyframe, frame node): that node's keyframe keys in index order, lanes over the candidates
//                   (best2_fold_warp); claims stay inside the node, so nodes are independent.
//   k_sbb_finish    one block per keyframe: the rotation histogram, ComputeThreeMaxima, the culling and the count.
#include <cfloat>
#include <climits>
#include <cmath>
#include <mutex>

#include "block_ops.cuh"
#include "host_call.h"
#include "match_fold.cuh"
#include "stream_scratch.h"
#include "vocabulary.h"

namespace sivo {
namespace {
constexpr int kMaxKeys = 16384;      // the block sorts keep pow2(keys) entries in shared memory
constexpr int kThLow = 50;           // ORBmatcher::TH_LOW
constexpr int kHisto = 30;           // ORBmatcher::HISTO_LENGTH
constexpr int kWarpThreads = 256, kWarps = kWarpThreads / 32;
constexpr int kBlockThreads = 1024;
constexpr int kChunk = 64;           // keyframes per launch (their table travels as a kernel parameter)
constexpr unsigned long long kNone = ~0ull;

int pow2_at_least(int n) {
  int p = 1;
  while (p < n) p <<= 1;
  return p;
}

// ascending bitonic sort of s[0 .. P), P a power of two, by the whole block
template <class T> __device__ void block_sort(T* s, int P) {
  __syncthreads();
  for (int k = 2; k <= P; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < P; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const T a = s[i], b = s[ixj];
          if ((a > b) == ((i & k) == 0)) { s[i] = b; s[ixj] = a; }
        }
      }
      __syncthreads();
    }
}

// ---------------------------------------------------------------------------------------------------------------- transform
__global__ void __launch_bounds__(kWarpThreads) k_bow_descend(const VocView v, const uint4* __restrict__ desc, const int* __restrict__ keep_idx,
                                                            const long long* __restrict__ n_keep, int cap, int nid_level, int* __restrict__ node,
                                                            int* __restrict__ word) {
  const int j = blockIdx.x * kWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int n = clamp_count(*n_keep, cap);
  if (j >= n) return;
  const int k = keep_idx ? keep_idx[j] : j;
  int out_node = -1, out_word = -1;
  if (k >= 0 && k < cap) {
    const uint4 q0 = desc[2 * k], q1 = desc[2 * k + 1];
    int id = 0, level = 0, nid = 0;
    bool nid_set = nid_level <= 0;
    int b = v.child_off[0], e = v.child_off[1];
    do {
      ++level;
      unsigned long long best = kNone;
      for (int c = b + lane; c < e; c += 32) {
        const int ch = v.children[c];
        const int d = descriptor_distance(q0, q1, v.desc[2 * ch], v.desc[2 * ch + 1]);
        best = min(best, (static_cast<unsigned long long>(d) << 32) | static_cast<unsigned>(c - b));
      }
#pragma unroll
      for (int o = 16; o; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
      id = v.children[b + static_cast<int>(best & 0xffffffffu)];
      if (level == nid_level) { nid = id; nid_set = true; }
      b = v.child_off[id];
      e = v.child_off[id + 1];
    } while (e > b);
    if (!nid_set) nid = id;  // a leaf above nid_level: the leaf itself
    const int w = v.node_word[id];
    if (v.word_weight[w] > 0.0) { out_node = nid; out_word = w; }
  }
  if (lane == 0) {
    if (node) node[j] = out_node;
    word[j] = out_word;
  }
}

__global__ void __launch_bounds__(kBlockThreads) k_bow_vector(const VocView v, const int* __restrict__ word, const long long* __restrict__ n_keep,
                                                              int cap, int* __restrict__ bow_word, double* __restrict__ bow_weight,
                                                              long long* __restrict__ bow_len) {
  extern __shared__ __align__(8) unsigned char smem[];
  double* val = reinterpret_cast<double*>(smem);  // cap doubles, then the sort's pow2 words (vector_smem)
  unsigned* s = reinterpret_cast<unsigned*>(val + cap);
  __shared__ int warp_count[kBlockThreads / 32];
  __shared__ double norm_s;
  const int tid = threadIdx.x;
  const int n = clamp_count(*n_keep, cap);
  if (n < 0) {
    if (tid == 0 && bow_len) *bow_len = -1;
    return;
  }
  int P = 1;
  while (P < n) P <<= 1;
  for (int i = tid; i < P; i += kBlockThreads) s[i] = i < n && word[i] >= 0 ? static_cast<unsigned>(word[i]) : 0xffffffffu;
  block_sort(s, P);
  const bool tf = v.weighting == SIVO_WEIGHTING_TF_IDF || v.weighting == SIVO_WEIGHTING_TF;
  int m = 0;  // BowVector entries so far
  for (int c0 = 0; c0 < n; c0 += kBlockThreads) {
    const int i = c0 + tid;
    const bool start = i < n && s[i] != 0xffffffffu && (i == 0 || s[i - 1] != s[i]);
    int total;
    const int rank = block_rank<kBlockThreads>(start, warp_count, &total);
    if (start) {
      const int pos = m + rank;
      int e = i + 1;
      while (e < n && s[e] == s[i]) ++e;
      const double w = v.word_weight[s[i]];
      double x = w;  // addWeight: w, then += w per further feature; addIfNotExist: the first feature's w
      if (tf)
        for (int r = i + 1; r < e; ++r) x += w;
      val[pos] = x;
      if (bow_word) bow_word[pos] = static_cast<int>(s[i]);
    }
    m += total;
    __syncthreads();
  }
  const bool must = v.scoring != SIVO_SCORING_DOT_PRODUCT;
  if (!must) {
    if (tf)
      for (int p = tid; p < m; p += kBlockThreads) val[p] /= static_cast<double>(m);
  } else {
    if (tid == 0) {
      double norm = 0.0;
      if (v.scoring == SIVO_SCORING_L2_NORM) {
        for (int p = 0; p < m; ++p) norm += val[p] * val[p];
        norm = sqrt(norm);
      } else {
        for (int p = 0; p < m; ++p) norm += fabs(val[p]);
      }
      norm_s = norm;
    }
    __syncthreads();
    const double norm = norm_s;
    if (norm > 0.0)
      for (int p = tid; p < m; p += kBlockThreads) val[p] /= norm;
  }
  __syncthreads();
  if (bow_weight)
    for (int p = tid; p < m; p += kBlockThreads) bow_weight[p] = val[p];
  if (tid == 0 && bow_len) *bow_len = m;
}

// ---------------------------------------------------------------------------------------------------------------- SearchByBoW
struct SbbKf {
  const sivo_keypoint* kps;
  const uint4* desc;
  const int* node;
  const int* point;
  const long long* count;
  int cap;  // the count's clamp
};

struct SbbChunk {
  SbbKf kf[kChunk];
  int n, base;
};

struct SbbFrame {
  const sivo_keypoint* kps;
  const uint4* desc;
  const int* keep_idx;
  const long long* n_keep;
  const int* node;
  int cap;  // keys per frame array and the stride of match's rows
  float nnratio;
  int check;
};

__device__ __forceinline__ int frame_key(const SbbFrame& f, int j) { return f.keep_idx ? f.keep_idx[j] : j; }

__global__ void __launch_bounds__(kBlockThreads) k_sbb_sort(const SbbFrame f, unsigned long long* __restrict__ sorted) {
  extern __shared__ __align__(8) unsigned char smem[];
  unsigned long long* s = reinterpret_cast<unsigned long long*>(smem);
  const int n = clamp_count(*f.n_keep, f.cap);
  if (n <= 0) return;
  int P = 1;
  while (P < n) P <<= 1;
  for (int i = threadIdx.x; i < P; i += kBlockThreads) {
    unsigned long long key = kNone;
    if (i < n) {
      const int k = frame_key(f, i), nd = f.node[i];
      if (k >= 0 && k < f.cap && nd >= 0 && angle_ok(f.kps[k].angle))
        key = (static_cast<unsigned long long>(nd) << 32) | static_cast<unsigned>(i);
    }
    s[i] = key;
  }
  block_sort(s, P);
  for (int i = threadIdx.x; i < n; i += kBlockThreads) sorted[i] = s[i];
}

// match rows of the keyframes this chunk searches start empty (vpMapPointMatches); rows of an affected keyframe are left alone
__global__ void k_sbb_init(const SbbFrame f, const SbbChunk c, int* __restrict__ match) {
  const int k = blockIdx.y;
  if (*f.n_keep < 0 || *c.kf[k].count < 0) return;
  int* row = match + static_cast<size_t>(c.base + k) * f.cap;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < f.cap; j += gridDim.x * blockDim.x) row[j] = -1;
}

__global__ void __launch_bounds__(kWarpThreads) k_sbb_walk(const SbbFrame f, const SbbChunk c, const unsigned long long* __restrict__ sorted,
                                                          int* __restrict__ match, uint8_t* __restrict__ bins) {
  const int w = blockIdx.x * kWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31, k = blockIdx.y;
  const int n = clamp_count(*f.n_keep, f.cap);
  const SbbKf& kf = c.kf[k];
  const int nk = clamp_count(*kf.count, kf.cap);
  if (n < 0 || nk < 0 || w >= n) return;
  const unsigned long long key = sorted[w];
  if (key == kNone) return;
  const unsigned v = static_cast<unsigned>(key >> 32);
  if (w > 0 && static_cast<unsigned>(sorted[w - 1] >> 32) == v) return;  // not the first key of its node
  int e = w + 1;  // the node's keys are sorted[w .. e)
  for (;; e += 32) {
    const int g = e + lane;
    const unsigned out = __ballot_sync(0xffffffffu, g >= n || static_cast<unsigned>(sorted[g < n ? g : 0] >> 32) != v);
    if (out) { e += __ffs(out) - 1; break; }
  }
  int* row = match + static_cast<size_t>(c.base + k) * f.cap;
  uint8_t* brow = bins + static_cast<size_t>(c.base + k) * f.cap;
  for (int i0 = 0; i0 < nk; i0 += 32) {
    const int i = i0 + lane;
    const bool ok = i < nk && kf.node[i] == static_cast<int>(v) && kf.point[i] >= 0 && angle_ok(kf.kps[i].angle);
    unsigned todo = __ballot_sync(0xffffffffu, ok);
    while (todo) {
      const int ii = i0 + __ffs(todo) - 1;
      todo &= todo - 1u;
      const uint4 q0 = kf.desc[2 * ii], q1 = kf.desc[2 * ii + 1];
      Best2 b;
      for (int g0 = w; g0 < e; g0 += 32) {
        const int g = g0 + lane;
        int d = 256, j = -1;
        if (g < e) {
          j = static_cast<int>(sorted[g] & 0xffffffffu);
          if (row[j] < 0) {
            const int fk = frame_key(f, j);
            d = descriptor_distance(q0, q1, f.desc[2 * fk], f.desc[2 * fk + 1]);
          }
        }
        best2_fold_warp(b, d, j, 0, min(32, e - g0));
      }
      if (b.dist <= kThLow && static_cast<float>(b.dist) < f.nnratio * static_cast<float>(b.dist2)) {
        if (lane == 0) {
          row[b.idx] = kf.point[ii];
          if (f.check) {
            float rot = kf.kps[ii].angle - f.kps[frame_key(f, b.idx)].angle;
            if (rot < 0.0f) rot += 360.0f;
            int bin = static_cast<int>(roundf(rot * (1.0f / kHisto)));
            if (bin == kHisto) bin = 0;
            brow[b.idx] = static_cast<uint8_t>(bin);
          }
        }
        __syncwarp();  // the claim is seen by every lane before the next keyframe key
      }
    }
  }
}

__global__ void __launch_bounds__(kWarpThreads) k_sbb_finish(const SbbFrame f, const SbbChunk c, int* __restrict__ match,
                                                            const uint8_t* __restrict__ bins, long long* __restrict__ n_matches) {
  __shared__ int hist[kHisto];
  __shared__ int keep[3];
  __shared__ int warp_sum[kWarps];
  const int k = blockIdx.x, tid = threadIdx.x;
  const int n = clamp_count(*f.n_keep, f.cap);
  if (n < 0 || *c.kf[k].count < 0) {
    if (tid == 0) n_matches[c.base + k] = -1;
    return;
  }
  int* row = match + static_cast<size_t>(c.base + k) * f.cap;
  const uint8_t* brow = bins + static_cast<size_t>(c.base + k) * f.cap;
  if (f.check) {
    if (tid < kHisto) hist[tid] = 0;
    __syncthreads();
    for (int j = tid; j < n; j += kWarpThreads)
      if (row[j] >= 0) atomicAdd(&hist[brow[j]], 1);
    __syncthreads();
    if (tid == 0) three_maxima(hist, kHisto, keep);
    __syncthreads();
    for (int j = tid; j < n; j += kWarpThreads)
      if (row[j] >= 0 && brow[j] != keep[0] && brow[j] != keep[1] && brow[j] != keep[2]) row[j] = -1;
    __syncthreads();
  }
  // each accepted match claimed a distinct frame key and each culled one was decremented once: the count is what remains
  int cnt = 0;
  for (int j = tid; j < n; j += kWarpThreads) cnt += row[j] >= 0;
#pragma unroll
  for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if ((tid & 31) == 0) warp_sum[tid >> 5] = cnt;
  __syncthreads();
  if (tid == 0) {
    int t = 0;
    for (int i = 0; i < kWarps; ++i) t += warp_sum[i];
    n_matches[c.base + k] = t;
  }
}

// ---------------------------------------------------------------------------------------------------------------- launches
size_t vector_smem(int cap) { return static_cast<size_t>(cap) * sizeof(double) + static_cast<size_t>(pow2_at_least(cap)) * sizeof(unsigned); }
size_t sort_smem(int cap) { return static_cast<size_t>(pow2_at_least(cap)) * sizeof(unsigned long long); }

// the block sorts' shared memory at the largest capacity, opted into once per device (the current one)
void ensure_smem_limits() {
  static std::mutex mu;
  static std::vector<int> done;
  int dev = 0;
  SIVO_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(mu);
  if (std::find(done.begin(), done.end(), dev) != done.end()) return;
  SIVO_CUDA(cudaFuncSetAttribute(k_bow_vector, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(vector_smem(kMaxKeys))));
  SIVO_CUDA(cudaFuncSetAttribute(k_sbb_sort, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(sort_smem(kMaxKeys))));
  done.push_back(dev);
}

void check_cap(int cap, const char* what) {
  if (cap > kMaxKeys) fail(SIVO_ERANGE, "%s: %d keys, at most %d", what, cap, kMaxKeys);
}

void launch_bow(const Vocabulary& voc, const uint8_t* desc, const int* keep_idx, const long long* n_keep, int cap, int levelsup, int* node,
                int* word, int* bow_word, double* bow_weight, long long* bow_len, cudaStream_t s) {
  const VocView v = voc.view();
  const int c = std::max(cap, 1);
  k_bow_descend<<<ceil_div(c, kWarps), kWarpThreads, 0, s>>>(v, reinterpret_cast<const uint4*>(desc), keep_idx, n_keep, cap,
                                                             voc.L - levelsup, node, word);
  SIVO_CUDA(cudaGetLastError());
  ensure_smem_limits();
  k_bow_vector<<<1, kBlockThreads, vector_smem(c), s>>>(v, word, n_keep, cap, bow_word, bow_weight, bow_len);
  SIVO_CUDA(cudaGetLastError());
}

void launch_sbb(const SbbFrame& f, const SbbKf* kfs, int n_kf, unsigned long long* sorted, uint8_t* bins, int* match, long long* n_matches,
                cudaStream_t s) {
  const int c = std::max(f.cap, 1);
  ensure_smem_limits();
  k_sbb_sort<<<1, kBlockThreads, sort_smem(c), s>>>(f, sorted);
  SIVO_CUDA(cudaGetLastError());
  for (int base = 0; base < n_kf; base += kChunk) {
    SbbChunk ch{};
    ch.base = base;
    ch.n = std::min(kChunk, n_kf - base);
    for (int i = 0; i < ch.n; ++i) ch.kf[i] = kfs[base + i];
    k_sbb_init<<<dim3(ceil_div(c, kWarpThreads), ch.n), kWarpThreads, 0, s>>>(f, ch, match);
    SIVO_CUDA(cudaGetLastError());
    k_sbb_walk<<<dim3(ceil_div(c, kWarps), ch.n), kWarpThreads, 0, s>>>(f, ch, sorted, match, bins);
    SIVO_CUDA(cudaGetLastError());
    k_sbb_finish<<<ch.n, kWarpThreads, 0, s>>>(f, ch, match, bins, n_matches);
    SIVO_CUDA(cudaGetLastError());
  }
}

void check_sbb_args(int n_kf, const sivo_keyframe_keys* kfs, const int* const* kf_point, float nnratio) {
  if (n_kf < 0) fail(SIVO_EINVAL, "search_by_bow: n_kf %d < 0", n_kf);
  if (n_kf > 0 && (!kfs || !kf_point)) fail(SIVO_EINVAL, "search_by_bow: null keyframes");
  if (!std::isfinite(nnratio)) fail(SIVO_EINVAL, "search_by_bow: nnratio not finite");
  for (int k = 0; k < n_kf; ++k)
    if (!kfs[k].count) fail(SIVO_EINVAL, "search_by_bow: keyframe %d has no count", k);
}
}  // namespace

void compute_bow_device(const Vocabulary& voc, const Orb& left, const uint8_t* desc, const int* keep_idx, const long long* n_keep,
                        int levelsup, int* node, int* word, int* bow_word, double* bow_weight, long long* bow_len, cudaStream_t s) {
  if (levelsup < 0) fail(SIVO_EINVAL, "compute_bow: levelsup %d < 0", levelsup);
  if (voc.device != left.device()) fail(SIVO_EINVAL, "compute_bow: the vocabulary is on device %d, the extractor on %d", voc.device, left.device());
  const int cap = left.capacity();
  check_cap(cap, "compute_bow");
  s = left.enter(s);
  const size_t c = std::max(cap, 1);
  StreamScratch sc(word ? 0 : StreamScratch::bytes<int>(c), s);
  launch_bow(voc, desc, keep_idx, n_keep, cap, levelsup, node, word ? word : sc.take<int>(c), bow_word, bow_weight, bow_len, s);
}

void compute_bow_host(const Vocabulary& voc, const uint8_t* desc, int n, int levelsup, int* node, int* word, int* bow_word,
                      double* bow_weight, int* bow_len) {
  if (levelsup < 0) fail(SIVO_EINVAL, "compute_bow: levelsup %d < 0", levelsup);
  if (n < 0 || (n > 0 && !desc)) fail(SIVO_EINVAL, "compute_bow: null descriptors or n < 0");
  check_cap(n, "compute_bow");
  HostCall& hc = host_call();
  hc.begin(voc.device);
  const long long nn = n;
  const uint8_t* d_desc = hc.upload(desc, 32 * static_cast<size_t>(n));
  const long long* d_n = hc.upload(&nn, 1);
  int* d_node = hc.take<int>(n);
  int* d_word = hc.take<int>(n);
  int* d_bw = hc.take<int>(n);
  double* d_bwt = hc.take<double>(n);
  long long* d_len = hc.take<long long>(1);
  launch_bow(voc, d_desc, nullptr, d_n, n, levelsup, d_node, d_word, d_bw, d_bwt, d_len, hc.stream);
  long long len = 0;
  hc.download(&len, d_len, 1);
  hc.download(node, d_node, n);
  hc.download(word, d_word, n);
  hc.sync();
  hc.download(bow_word, d_bw, static_cast<size_t>(len));
  hc.download(bow_weight, d_bwt, static_cast<size_t>(len));
  hc.sync();
  if (bow_len) *bow_len = static_cast<int>(len);
}

void search_by_bow_device(const Orb& left, const sivo_keypoint* kps, const uint8_t* desc, const int* keep_idx, const long long* n_keep,
                          const int* node, const sivo_keyframe_keys* kfs, const int* const* kf_point, int n_kf, float nnratio, int check,
                          int* match, long long* n_matches, cudaStream_t s) {
  check_sbb_args(n_kf, kfs, kf_point, nnratio);
  const int cap = left.capacity();
  check_cap(cap, "search_by_bow");
  std::vector<SbbKf> t(n_kf);
  for (int k = 0; k < n_kf; ++k) {
    if (!kfs[k].kps || !kfs[k].desc || !kfs[k].node || !kf_point[k]) fail(SIVO_EINVAL, "search_by_bow: null array in keyframe %d", k);
    t[k] = SbbKf{kfs[k].kps, reinterpret_cast<const uint4*>(kfs[k].desc), kfs[k].node, kf_point[k], kfs[k].count, cap};
  }
  s = left.enter(s);
  const SbbFrame f{kps, reinterpret_cast<const uint4*>(desc), keep_idx, n_keep, node, cap, nnratio, check ? 1 : 0};
  // the frame's sorted keys and one rotation bin per (keyframe, frame key)
  const size_t c = std::max(cap, 1), n_bins = static_cast<size_t>(n_kf) * cap;
  StreamScratch sc(StreamScratch::bytes<unsigned long long>(c) + n_bins, s);
  unsigned long long* sorted = sc.take<unsigned long long>(c);
  launch_sbb(f, t.data(), n_kf, sorted, sc.take<uint8_t>(n_bins), match, n_matches, s);
}

void search_by_bow_host(const Orb& left, const sivo_keypoint* kps, const uint8_t* desc, const int* node, int n,
                        const sivo_keyframe_keys* kfs, const int* const* kf_point, int n_kf, float nnratio, int check, int* match,
                        long long* n_matches) {
  check_sbb_args(n_kf, kfs, kf_point, nnratio);
  if (n < 0 || (n > 0 && (!kps || !desc || !node))) fail(SIVO_EINVAL, "search_by_bow: null frame array or n < 0");
  if (n_kf > 0 && !n_matches) fail(SIVO_EINVAL, "search_by_bow: null n_matches");
  if (n_kf > 0 && n > 0 && !match) fail(SIVO_EINVAL, "search_by_bow: null match");
  check_cap(n, "search_by_bow");
  for (int j = 0; j < n; ++j)
    if (!angle_ok(kps[j].angle)) fail(SIVO_ERANGE, "search_by_bow: frame key %d angle %g outside [0, 360]", j, kps[j].angle);
  HostCall& hc = host_call();
  hc.begin(left.device());
  std::vector<SbbKf> t(n_kf);
  for (int k = 0; k < n_kf; ++k) {
    const long long c = *kfs[k].count;
    const int m = static_cast<int>(std::max(c, 0ll));
    if (c > kMaxKeys) fail(SIVO_ERANGE, "search_by_bow: keyframe %d has %lld keys, at most %d", k, c, kMaxKeys);
    if (m > 0 && (!kfs[k].kps || !kfs[k].desc || !kfs[k].node || !kf_point[k])) fail(SIVO_EINVAL, "search_by_bow: null array in keyframe %d", k);
    for (int i = 0; i < m; ++i)
      if (!angle_ok(kfs[k].kps[i].angle))
        fail(SIVO_ERANGE, "search_by_bow: keyframe %d key %d angle %g outside [0, 360]", k, i, kfs[k].kps[i].angle);
    t[k] = SbbKf{hc.upload(kfs[k].kps, m), reinterpret_cast<const uint4*>(hc.upload(kfs[k].desc, 32 * static_cast<size_t>(m))),
                 hc.upload(kfs[k].node, m), hc.upload(kf_point[k], m), hc.upload(kfs[k].count, 1), m};
  }
  const long long nn = n;
  const SbbFrame f{hc.upload(kps, n), reinterpret_cast<const uint4*>(hc.upload(desc, 32 * static_cast<size_t>(n))), nullptr, hc.upload(&nn, 1),
                   hc.upload(node, n), n, nnratio, check ? 1 : 0};
  const size_t cells = static_cast<size_t>(n_kf) * n;
  unsigned long long* d_sorted = hc.take<unsigned long long>(n);
  uint8_t* d_bins = hc.take<uint8_t>(cells);
  int* d_match = hc.take<int>(cells);
  long long* d_nm = hc.take<long long>(n_kf);
  launch_sbb(f, t.data(), n_kf, d_sorted, d_bins, d_match, d_nm, hc.stream);
  hc.download(n_matches, d_nm, n_kf);
  hc.sync();
  // rows of an affected keyframe were not written: leave the caller's memory alone there too
  for (int k = 0; k < n_kf; ++k)
    if (n_matches[k] >= 0) hc.download(match + static_cast<size_t>(k) * n, d_match + static_cast<size_t>(k) * n, n);
  hc.sync();
}

}  // namespace sivo
