// DistributeOctTree (src/orbslam/ORBextractor.cc:544-750, ExtractorNode::DivideNode :488-542) on the device: one thread
// block per pyramid level, the whole tree in shared memory.  Same function as the host restatement `orb_distribute`
// (orb_host.cu) -- same node order, same documented tie rule (creation order instead of the reference's heap-pointer order in
// the last round) -- so the selected keypoints and their ORDER are identical; tests compare the two on random inputs and on
// whole images.  With the tree on the device the extractor has no host round trip: pyramid -> FAST -> cells -> tree ->
// describe is one asynchronous chain of launches (the host path remains for inputs that exceed the shared-memory caps).
//
// Representation.  Keys stay in place; `perm` holds key indices and every node owns a contiguous range of it (a split is a
// stable 4-way partition of that range, as in the host version).  The reference's std::list is an ARRAY in list order:
// a regular round visits the list front to back, replaces every splittable node by its non-empty children (each
// `push_front`), and leaves the others in place, so
//     new list = reverse(children in creation order) ++ (unsplit nodes in their old order),
// which a prefix sum over the old list computes in parallel (one warp per node does the partitions).  The last phase (largest
// nodes first, one at a time, stop as soon as the target is reached) is sequential by nature: one warp runs it, pushing
// children on a `front` stack (list = reverse(front) ++ base) and clearing the parents' alive flags.
#include <cuda_runtime.h>

#include <cstdint>

#include "orb.h"

namespace sivo {

namespace {

constexpr int kTreeThreads = 512, kTreeWarps = kTreeThreads / 32;

struct TreeNode {
  short ulx, uly, urx, bry;
  unsigned short begin, count, seq;
  unsigned char no_more, alive;
};

struct TreeSmem {
  unsigned short kx[kTreeKeyCap], ky[kTreeKeyCap];
  unsigned char kr[kTreeKeyCap];
  unsigned short perm[kTreeKeyCap], perm2[kTreeKeyCap];
  TreeNode node[kTreeNodeCap];
  unsigned short base[kTreeListCap], base2[kTreeListCap], front[kTreeListCap];
  unsigned short pend[kTreeListCap], pend2[kTreeListCap];   // splittable children in creation order (node ids)
  unsigned short seq2node[kTreeNodeCap];
  unsigned short cnt[kTreeListCap][4];                       // per list position: child sizes of this round's split
  unsigned int sortkey[kTreeListCap];
  int scan[kTreeWarps];
  int warp_cnt[kTreeWarps][16];
  int n_nodes, size, base_len, n_front, n_pend, n_pend2, seq, error, finish;
};

__device__ __forceinline__ int ceil_half(int d) { return (d + 1) >> 1; }  // ceil(d / 2.f) for d >= 0

// exclusive block scan of one int per thread (returns the prefix; *total = sum); all threads must call
__device__ int block_exscan(int v, int* scratch, int* total) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  __syncthreads();  // scratch may still be read from a previous call
  if (lane == 31) scratch[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    int w = lane < kTreeWarps ? scratch[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += t;
    }
    if (lane < kTreeWarps) scratch[lane] = w;
  }
  __syncthreads();
  const int warp_off = warp ? scratch[warp - 1] : 0;
  *total = scratch[kTreeWarps - 1];
  return warp_off + inc - v;
}

// One warp partitions node `id` (ExtractorNode::DivideNode): stable 4-way partition of its key range by quadrant
// (UL, UR, BL, BR = !(x < mx) + 2 * !(y < my)) into perm2, child sizes to out_cnt[4].  warp_commit() copies the range back to
// perm: a node that ends up NOT being split (last phase, past the cut-off) keeps its key order, which decides response ties.
__device__ void warp_partition(TreeSmem& s, int id, unsigned short* out_cnt) {
  const int lane = threadIdx.x & 31;
  const TreeNode nd = s.node[id];
  const int mx = nd.ulx + ceil_half(nd.urx - nd.ulx), my = nd.uly + ceil_half(nd.bry - nd.uly);
  int c[4] = {0, 0, 0, 0};
  for (int i0 = 0; i0 < nd.count; i0 += 32) {
    const int i = i0 + lane;
    int q = -1;
    if (i < nd.count) {
      const int k = s.perm[nd.begin + i];
      q = static_cast<int>(!(s.kx[k] < mx)) + 2 * static_cast<int>(!(s.ky[k] < my));
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) c[j] += __popc(__ballot_sync(0xffffffffu, q == j));
  }
  int off[4] = {0, c[0], c[0] + c[1], c[0] + c[1] + c[2]};
  for (int i0 = 0; i0 < nd.count; i0 += 32) {
    const int i = i0 + lane;
    int q = -1, k = 0;
    if (i < nd.count) {
      k = s.perm[nd.begin + i];
      q = static_cast<int>(!(s.kx[k] < mx)) + 2 * static_cast<int>(!(s.ky[k] < my));
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const unsigned b = __ballot_sync(0xffffffffu, q == j);
      if (q == j) s.perm2[nd.begin + off[j] + __popc(b & ((1u << lane) - 1u))] = static_cast<unsigned short>(k);
      off[j] += __popc(b);
    }
  }
  if (lane < 4) out_cnt[lane] = static_cast<unsigned short>(c[lane]);
  __syncwarp();
}
__device__ void warp_commit(TreeSmem& s, int id) {
  const int lane = threadIdx.x & 31;
  const int b = s.node[id].begin, n = s.node[id].count;
  for (int i = lane; i < n; i += 32) s.perm[b + i] = s.perm2[b + i];
  __syncwarp();
}

__device__ __forceinline__ TreeNode child_of(const TreeNode& p, int q, int start, int c) {
  const int mx = p.ulx + ceil_half(p.urx - p.ulx), my = p.uly + ceil_half(p.bry - p.uly);
  TreeNode ch;
  ch.ulx = static_cast<short>((q & 1) ? mx : p.ulx);
  ch.urx = static_cast<short>((q & 1) ? p.urx : mx);
  ch.uly = static_cast<short>((q & 2) ? my : p.uly);
  ch.bry = static_cast<short>((q & 2) ? p.bry : my);
  ch.begin = static_cast<unsigned short>(p.begin + start);
  ch.count = static_cast<unsigned short>(c);
  ch.seq = 0;
  ch.no_more = c == 1;
  ch.alive = 1;
  return ch;
}

// cand: packed x | y << 12 | response << 24 (k_cells), all levels, level l at [level_off[l], level_off[l + 1]).
// out_sel[l * kTreeSelCap + i]: packed candidate of the i-th retained keypoint of level l (list order); out_count[l].
// A level that does not fit the shared-memory caps sets bit l of *out_error (the host then takes its own path).
// Input either as the compacted candidate array (cand / level_off) or -- cell_items != nullptr -- straight from the per-cell lists
// k_cells wrote (cell c of the level holds cell_count[c] items at cell_items[c * kCellCap ...]; cells in row-major order, which is
// the reference's vToDistributeKeys order), sparing the scan / gather launches.
__global__ void __launch_bounds__(kTreeThreads, 1)
k_distribute(const uint32_t* __restrict__ cand, const int* __restrict__ level_off, const uint32_t* __restrict__ cell_items,
             const int* __restrict__ cell_count, OrbTreeParams prm, uint32_t* __restrict__ out_sel, int* __restrict__ out_count,
             int* __restrict__ out_error) {
  extern __shared__ __align__(16) uint8_t tree_raw[];
  TreeSmem& s = *reinterpret_cast<TreeSmem*>(tree_raw);
  const int l = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n_target = prm.n_target[l], n_ini = prm.n_ini[l];
  const float hx = prm.hx[l];
  int m;
  if (cell_items) {
    // exclusive scan of the level's cell counts (cells may outnumber the threads: strided passes), then one warp per cell
    const int c0 = prm.cell_begin[l], nc = prm.cell_end[l] - c0;
    int total = 0;
    bool too_many = false;
    for (int base_c = 0; base_c < nc; base_c += kTreeThreads) {
      const int c = base_c + tid;
      const int n = c < nc ? min(cell_count[c0 + c], kCellCap) : 0;
      int t;
      const int off = total + block_exscan(n, s.scan, &t);
      if (c < nc && c < kTreeNodeCap) s.seq2node[c] = static_cast<unsigned short>(min(off, 65535));  // scratch: the cell's offset
      total += t;
      if (nc > kTreeNodeCap) too_many = true;
    }
    m = total;
    if (m > kTreeKeyCap || too_many) {
      if (tid == 0) { out_count[l] = 0; atomicOr(out_error, 1 << l); }
      return;
    }
    __syncthreads();
    for (int c = warp; c < nc; c += kTreeWarps) {
      const int n = min(cell_count[c0 + c], kCellCap), off = s.seq2node[c];
      for (int i = lane; i < n; i += 32) {
        const uint32_t v = cell_items[static_cast<size_t>(c0 + c) * kCellCap + i];
        s.kx[off + i] = static_cast<unsigned short>(v & 0xFFF);
        s.ky[off + i] = static_cast<unsigned short>((v >> 12) & 0xFFF);
        s.kr[off + i] = static_cast<unsigned char>(v >> 24);
      }
    }
    __syncthreads();
  } else {
    const int b0 = level_off[l];
    m = level_off[l + 1] - b0;
    if (m > 0 && m <= kTreeKeyCap)
      for (int k = tid; k < m; k += kTreeThreads) {
        const uint32_t c = cand[b0 + k];
        s.kx[k] = static_cast<unsigned short>(c & 0xFFF);
        s.ky[k] = static_cast<unsigned short>((c >> 12) & 0xFFF);
        s.kr[k] = static_cast<unsigned char>(c >> 24);
      }
  }
  if (m <= 0) { if (tid == 0) out_count[l] = 0; return; }
  if (m > kTreeKeyCap || n_ini > 16 || n_target + 8 > kTreeSelCap) {
    if (tid == 0) { out_count[l] = 0; atomicOr(out_error, 1 << l); }
    return;
  }
  // ---- initial cells: stable counting sort by int(x / hx), clamped (ORBextractor.cc:551-575)
  if (tid < kTreeWarps * 16) (&s.warp_cnt[0][0])[tid] = 0;
  if (tid == 0) { s.error = 0; s.finish = 0; }
  __syncthreads();
  const int per_warp = (m + kTreeWarps - 1) / kTreeWarps;
  const int k_lo = min(m, warp * per_warp), k_hi = min(m, k_lo + per_warp);
  auto cell_of = [&](int k) {
    const int c = static_cast<int>(__fdiv_rn(static_cast<float>(s.kx[k]), hx));
    return c >= n_ini ? n_ini - 1 : c;
  };
  for (int k0 = k_lo; k0 < k_hi; k0 += 32) {
    const int k = k0 + lane;
    const int c = k < k_hi ? cell_of(k) : -1;
    for (int j = 0; j < n_ini; ++j) {
      const int n = __popc(__ballot_sync(0xffffffffu, c == j));
      if (lane == 0) s.warp_cnt[warp][j] += n;
    }
  }
  __syncthreads();
  if (tid == 0) {
    // nodes 0 .. n_ini - 1 in creation order (push_back); warp_cnt becomes the write cursor of each (warp, cell)
    int off = 0;
    for (int j = 0; j < n_ini; ++j) {
      TreeNode nd;
      nd.ulx = static_cast<short>(static_cast<int>(__fmul_rn(hx, static_cast<float>(j))));
      nd.urx = static_cast<short>(static_cast<int>(__fmul_rn(hx, static_cast<float>(j + 1))));
      nd.uly = 0;
      nd.bry = static_cast<short>(prm.height[l]);
      nd.begin = static_cast<unsigned short>(off);
      int c = 0;
      for (int w = 0; w < kTreeWarps; ++w) { const int t = s.warp_cnt[w][j]; s.warp_cnt[w][j] = off + c; c += t; }
      nd.count = static_cast<unsigned short>(c);
      nd.seq = 0;
      nd.no_more = c == 1;
      nd.alive = 1;
      s.node[j] = nd;
      off += c;
    }
    int sz = 0;
    for (int j = 0; j < n_ini; ++j) if (s.node[j].count > 0) s.base[sz++] = static_cast<unsigned short>(j);  // empty cells are erased
    s.size = s.base_len = sz;
    s.n_nodes = n_ini;
    s.seq = 0;
    s.n_front = 0;
    s.n_pend = 0;
  }
  __syncthreads();
  for (int k0 = k_lo; k0 < k_hi; k0 += 32) {
    const int k = k0 + lane;
    const int c = k < k_hi ? cell_of(k) : -1;
    for (int j = 0; j < n_ini; ++j) {
      const unsigned b = __ballot_sync(0xffffffffu, c == j);
      if (c == j) s.perm[s.warp_cnt[warp][j] + __popc(b & ((1u << lane) - 1u))] = static_cast<unsigned short>(k);
      __syncwarp();
      if (lane == 0) s.warp_cnt[warp][j] += __popc(b);
      __syncwarp();
    }
  }
  __syncthreads();

  // ---- regular rounds (:585-665)
  bool last_phase = false;
  for (int guard = 0; guard < 64; ++guard) {
    const int S = s.size;  // == base_len: the front stack is empty in this phase
    // (1) every splittable node of the list is partitioned, one warp per node
    for (int i = warp; i < S; i += kTreeWarps) {
      const int id = s.base[i];
      if (!s.node[id].no_more) { warp_partition(s, id, s.cnt[i]); warp_commit(s, id); }
    }
    __syncthreads();
    const int n_nodes0 = s.n_nodes, seq0 = s.seq;
    // (2) pass A: number of children this round creates (they go in front of the nodes that stay)
    int G = 0;
    for (int base_i = 0; base_i < S; base_i += kTreeThreads) {
      const int i = base_i + tid;
      int c = 0;
      if (i < S && !s.node[s.base[i]].no_more)
        for (int q = 0; q < 4; ++q) c += s.cnt[i][q] > 0;
      int t;
      block_exscan(c, s.scan, &t);
      G += t;
    }
    int n_keep_total = 0;
    if (n_nodes0 + G > kTreeNodeCap || G + S > kTreeListCap) {
      if (tid == 0) { atomicOr(out_error, 1 << l); out_count[l] = 0; }
      return;
    }
    // (3) pass B: children in creation order = list order of the parents, quadrant order within a parent
    int tot_ch = 0, tot_sp = 0;
    for (int base_i = 0; base_i < S; base_i += kTreeThreads) {
      const int i = base_i + tid;
      int nch = 0, nsp = 0, nkeep = 0, pid = 0;
      TreeNode par;
      bool split = false;
      if (i < S) {
        pid = s.base[i];
        par = s.node[pid];
        split = !par.no_more;
        if (split) for (int q = 0; q < 4; ++q) { nch += s.cnt[i][q] > 0; nsp += s.cnt[i][q] > 1; }
        else nkeep = 1;
      }
      int t_ch, t_sp, t_keep;
      const int e_ch = block_exscan(nch, s.scan, &t_ch);
      const int e_sp = block_exscan(nsp, s.scan, &t_sp);
      const int e_keep = block_exscan(nkeep, s.scan, &t_keep);
      if (i < S) {
        if (split) {
          int g = tot_ch + e_ch, sp = tot_sp + e_sp, start = 0;
          for (int q = 0; q < 4; ++q) {
            const int c = s.cnt[i][q];
            if (c) {
              TreeNode ch = child_of(par, q, start, c);
              const int cid = n_nodes0 + g;
              if (c > 1) {
                ch.seq = static_cast<unsigned short>(seq0 + sp + 1);
                s.seq2node[ch.seq] = static_cast<unsigned short>(cid);
                s.pend[sp] = static_cast<unsigned short>(cid);
                ++sp;
              }
              s.node[cid] = ch;
              s.base2[G - 1 - g] = static_cast<unsigned short>(cid);
              ++g;
            }
            start += c;
          }
          s.node[pid].alive = 0;
        } else {
          s.base2[G + n_keep_total + e_keep] = static_cast<unsigned short>(pid);
        }
      }
      tot_ch += t_ch; tot_sp += t_sp; n_keep_total += t_keep;
    }
    __syncthreads();
    const int S_new = G + n_keep_total;
    for (int i = tid; i < S_new; i += kTreeThreads) s.base[i] = s.base2[i];
    __syncthreads();
    if (tid == 0) {
      s.n_nodes = n_nodes0 + G;
      s.seq = seq0 + tot_sp;
      s.size = s.base_len = S_new;
      s.n_pend = tot_sp;
    }
    __syncthreads();
    if (S_new >= n_target || S_new == S) break;                           // (:659-662)
    if (S_new + 3 * tot_sp > n_target) { last_phase = true; break; }      // (:663)
  }

  // ---- last phase (:665-732): largest nodes first, one split at a time, until the target is reached.  Sequential in the
  // reference; here every node of the round is partitioned tentatively (in parallel, into perm2), the gains (children - 1) are
  // prefix-summed in processing order, the first position that reaches the target is the cut-off, and only the splits up to it
  // are committed -- children, creation sequence numbers and list positions follow from the same prefix sums.
  while (last_phase) {
    const int R = s.n_pend, prev = s.size;
    // processing order = descending (count, seq) (std::sort on (size, pointer) pairs in the reference; ties by creation order
    // here): rank sort, the keys are unique
    for (int i = tid; i < R; i += kTreeThreads)
      s.sortkey[i] = (static_cast<unsigned>(s.node[s.pend[i]].count) << 16) | s.node[s.pend[i]].seq;
    __syncthreads();
    for (int i = tid; i < R; i += kTreeThreads) {
      const unsigned key = s.sortkey[i];
      int larger = 0;
      for (int j = 0; j < R; ++j) larger += s.sortkey[j] > key;
      s.base2[larger] = s.pend[i];  // base2[p] = the p-th node to be processed
    }
    if (tid == 0) s.finish = R;  // cut-off position (exclusive bound on committed splits), lowered below
    __syncthreads();
    for (int p = warp; p < R; p += kTreeWarps) warp_partition(s, s.base2[p], s.cnt[p]);
    __syncthreads();
    // cut-off: first p with size + sum_{p' <= p} (children(p') - 1) >= target
    int run_gain = 0;
    for (int base_p = 0; base_p < R; base_p += kTreeThreads) {
      const int p2 = base_p + tid;
      int gain = 0;
      if (p2 < R) { for (int q = 0; q < 4; ++q) gain += s.cnt[p2][q] > 0; gain -= 1; }
      int t;
      const int exc = block_exscan(gain, s.scan, &t);
      if (p2 < R && prev + run_gain + exc + gain >= n_target) atomicMin(&s.finish, p2 + 1);
      run_gain += t;
    }
    __syncthreads();
    const int Cn = s.finish;  // splits 0 .. Cn-1 are committed
    const int n_nodes0 = s.n_nodes, seq0 = s.seq, nf0 = s.n_front;
    int tot_ch = 0, tot_sp = 0;
    bool overflow = false;
    for (int base_p = 0; base_p < Cn; base_p += kTreeThreads) {
      const int p2 = base_p + tid;
      int nch = 0, nsp = 0;
      if (p2 < Cn) for (int q = 0; q < 4; ++q) { nch += s.cnt[p2][q] > 0; nsp += s.cnt[p2][q] > 1; }
      int t_ch, t_sp;
      const int e_ch = block_exscan(nch, s.scan, &t_ch);
      const int e_sp = block_exscan(nsp, s.scan, &t_sp);
      if (n_nodes0 + tot_ch + t_ch > kTreeNodeCap || nf0 + tot_ch + t_ch > kTreeListCap || tot_sp + t_sp > kTreeListCap) overflow = true;
      if (p2 < Cn && !overflow) {
        const int pid = s.base2[p2];
        const TreeNode par = s.node[pid];
        int g = tot_ch + e_ch, sp = tot_sp + e_sp, start = 0;
        for (int q = 0; q < 4; ++q) {
          const int c = s.cnt[p2][q];
          if (c) {
            TreeNode ch = child_of(par, q, start, c);
            const int cid = n_nodes0 + g;
            if (c > 1) {
              ch.seq = static_cast<unsigned short>(seq0 + sp + 1);
              s.seq2node[ch.seq] = static_cast<unsigned short>(cid);
              s.pend2[sp] = static_cast<unsigned short>(cid);
              ++sp;
            }
            s.node[cid] = ch;
            s.front[nf0 + g] = static_cast<unsigned short>(cid);  // push_front, in processing order
            ++g;
          }
          start += c;
        }
        s.node[pid].alive = 0;  // erase
      }
      tot_ch += t_ch; tot_sp += t_sp;
    }
    __syncthreads();
    if (overflow) {
      if (tid == 0) { atomicOr(out_error, 1 << l); out_count[l] = 0; }
      return;
    }
    for (int p = warp; p < Cn; p += kTreeWarps) warp_commit(s, s.base2[p]);  // the parents' ranges, now their children's
    const int size_new = prev + tot_ch - Cn;
    __syncthreads();
    for (int i = tid; i < tot_sp; i += kTreeThreads) s.pend[i] = s.pend2[i];
    if (tid == 0) {
      s.n_nodes = n_nodes0 + tot_ch;
      s.seq = seq0 + tot_sp;
      s.n_front = nf0 + tot_ch;
      s.size = size_new;
      s.n_pend = tot_sp;
    }
    __syncthreads();
    if (size_new >= n_target || size_new == prev) break;
  }

  // ---- output (:735-748): list = reverse(front) ++ base, alive nodes only; per node the first key with the largest response
  const int nf = s.n_front, E = nf + s.base_len;
  int written = 0;
  for (int base_e = 0; base_e < E; base_e += kTreeThreads) {
    const int e = base_e + tid;
    int id = -1;
    if (e < E) {
      id = e < nf ? s.front[nf - 1 - e] : s.base[e - nf];
      if (!s.node[id].alive) id = -1;
    }
    int t;
    const int pos = written + block_exscan(id >= 0 ? 1 : 0, s.scan, &t);
    if (id >= 0 && pos < kTreeSelCap) {
      const TreeNode nd = s.node[id];
      int best = s.perm[nd.begin];
      for (int k = 1; k < nd.count; ++k) {
        const int kk = s.perm[nd.begin + k];
        if (s.kr[kk] > s.kr[best]) best = kk;
      }
      out_sel[l * kTreeSelCap + pos] = static_cast<uint32_t>(s.kx[best]) | (static_cast<uint32_t>(s.ky[best]) << 12) |
                                       (static_cast<uint32_t>(s.kr[best]) << 24);
    }
    written += t;
  }
  if (tid == 0) {
    if (written > kTreeSelCap) { atomicOr(out_error, 1 << l); written = 0; }
    out_count[l] = written;
  }
}

}  // namespace

void orb_tree_configure() {
  static_assert(sizeof(TreeSmem) <= 227 * 1024, "the tree must fit one CTA's shared memory");
  SIVO_CUDA(cudaFuncSetAttribute(k_distribute, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(sizeof(TreeSmem))));
}

void orb_launch_distribute(const uint32_t* cand, const int* level_off, const uint32_t* cell_items, const int* cell_count,
                           const OrbTreeParams& prm, int nlevels, uint32_t* sel_packed, int* level_count, int* error, cudaStream_t s) {
  k_distribute<<<nlevels, kTreeThreads, sizeof(TreeSmem), s>>>(cand, level_off, cell_items, cell_count, prm, sel_packed, level_count, error);
  SIVO_CUDA(cudaGetLastError());
}

}  // namespace sivo
