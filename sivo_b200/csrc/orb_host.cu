// Host side of the ORB operator: constructor tables, the per-level cell grid, the host quad tree (the fallback for levels beyond
// the device tree's caps), and the device schedule
//   device tree: [pyramid, cells, blur, quad tree, angle+rBRIEF] -> D2H
//   host tree:   [pyramid, cells, compact, blur] -> candidates D2H -> quad tree -> selection H2D -> [angle+rBRIEF] -> D2H.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <mutex>
#include <string>

#include "orb.h"

namespace sivo {

// ---------------------------------------------------------------- ORBextractor::ORBextractor (:412-475)
OrbTables orb_make_tables(int nfeatures, float scale_factor, int nlevels) {
  OrbTables t;
  const double sf = static_cast<double>(scale_factor);  // the member is a double initialised from the float argument
  t.scale.assign(nlevels, 1.f);
  t.sigma2.assign(nlevels, 1.f);
  for (int i = 1; i < nlevels; ++i) {
    t.scale[i] = static_cast<float>(t.scale[i - 1] * sf);
    t.sigma2[i] = t.scale[i] * t.scale[i];
  }
  t.inv_scale.resize(nlevels);
  t.inv_sigma2.resize(nlevels);
  for (int i = 0; i < nlevels; ++i) {
    t.inv_scale[i] = 1.0f / t.scale[i];
    t.inv_sigma2[i] = 1.0f / t.sigma2[i];
  }
  t.per_level.assign(nlevels, 0);
  const float factor = static_cast<float>(1.0f / sf);
  float desired = nfeatures * (1 - factor) / (1 - static_cast<float>(std::pow(static_cast<double>(factor), static_cast<double>(nlevels))));
  int sum = 0;
  for (int l = 0; l < nlevels - 1; ++l) {
    t.per_level[l] = static_cast<int>(std::nearbyint(desired));
    sum += t.per_level[l];
    desired *= factor;
  }
  t.per_level[nlevels - 1] = std::max(nfeatures - sum, 0);
  // end of each row of the radius-15 disc
  const float hs = kHalfPatch * std::sqrt(2.f) / 2;
  const int vmax = static_cast<int>(std::floor(hs + 1));
  const int vmin = static_cast<int>(std::ceil(hs));
  const double hp2 = kHalfPatch * kHalfPatch;
  for (int v = 0; v <= kHalfPatch; ++v) t.umax[v] = 0;
  for (int v = 0; v <= vmax; ++v) t.umax[v] = static_cast<int>(std::nearbyint(std::sqrt(hp2 - v * v)));
  for (int v = kHalfPatch, v0 = 0; v >= vmin; --v) {
    while (t.umax[v0] == t.umax[v0 + 1]) ++v0;
    t.umax[v] = v0;
    ++v0;
  }
  return t;
}

// ---------------------------------------------------------------- DistributeOctTree (:544-750)
namespace {
struct QNode {
  int ulx, uly, urx, bry;
  int begin = 0, count = 0;  // this node's keys: perm[begin, begin + count), in the reference's vKeys order
  bool no_more = false;
  int prev = -1, next = -1;  // intrusive list links (arena indices)
  int seq = 0;               // creation order among splittable nodes: the documented tie-break
};

struct QList {
  std::vector<QNode> arena;
  int head = -1, tail = -1, size = 0;
  int make() { arena.emplace_back(); return static_cast<int>(arena.size()) - 1; }
  void push_front(int i) {
    arena[i].prev = -1;
    arena[i].next = head;
    if (head >= 0) arena[head].prev = i; else tail = i;
    head = i;
    ++size;
  }
  void push_back(int i) {
    arena[i].next = -1;
    arena[i].prev = tail;
    if (tail >= 0) arena[tail].next = i; else head = i;
    tail = i;
    ++size;
  }
  int erase(int i) {  // returns the successor
    int p = arena[i].prev, n = arena[i].next;
    if (p >= 0) arena[p].next = n; else head = n;
    if (n >= 0) arena[n].prev = p; else tail = p;
    --size;
    return n;
  }
};
}  // namespace

// Keys live in one permutation array; a node owns a contiguous range of it and a split is a stable 4-way partition of
// that range (children keep the parent's key order, as the reference's per-child push_back does), so the tree allocates
// nothing per node.
std::vector<int> orb_distribute(const float* xs, const float* ys, const float* resp, int n, int min_x, int max_x, int min_y,
                                int max_y, int n_target) {
  std::vector<int> result;
  if (n <= 0) return result;
  static thread_local QList L;
  static thread_local std::vector<int> perm, scratch, ini, pending, round;
  static thread_local std::vector<uint8_t> quad;
  L.arena.clear();
  L.head = L.tail = -1;
  L.size = 0;
  L.arena.reserve(static_cast<size_t>(n) * 4 + 64);
  perm.resize(n);
  scratch.resize(n);
  quad.resize(n);
  int n_ini = static_cast<int>(std::round(static_cast<float>(max_x - min_x) / (max_y - min_y)));
  if (n_ini < 1) n_ini = 1;  // the reference divides by zero here for tall images; not reachable on this path
  const float hx = static_cast<float>(max_x - min_x) / n_ini;
  ini.assign(n_ini, 0);
  for (int i = 0; i < n_ini; ++i) {
    int id = L.make();
    QNode& nd = L.arena[id];
    nd.ulx = static_cast<int>(hx * static_cast<float>(i));
    nd.urx = static_cast<int>(hx * static_cast<float>(i + 1));
    nd.uly = 0;
    nd.bry = max_y - min_y;
    L.push_back(id);
    ini[i] = id;
  }
  // stable counting sort of the keys by initial cell
  for (int k = 0; k < n; ++k) {
    int cell = static_cast<int>(xs[k] / hx);
    if (cell >= n_ini) cell = n_ini - 1;
    scratch[k] = cell;
    ++L.arena[ini[cell]].count;
  }
  for (int i = 0, off = 0; i < n_ini; ++i) {
    QNode& nd = L.arena[ini[i]];
    nd.begin = off;
    off += nd.count;
    nd.count = 0;
  }
  for (int k = 0; k < n; ++k) {
    QNode& nd = L.arena[ini[scratch[k]]];
    perm[nd.begin + nd.count++] = k;
  }
  for (int i = L.head; i >= 0;) {
    QNode& nd = L.arena[i];
    if (nd.count == 1) { nd.no_more = true; i = nd.next; }
    else if (nd.count == 0) i = L.erase(i);
    else i = nd.next;
  }
  int seq = 0;
  pending.clear();  // splittable children created in the current round
  auto split = [&](int id, int& n_expand) {
    // ExtractorNode::DivideNode (:488-542)
    const QNode parent = L.arena[id];  // copy: the arena may reallocate below
    const int half_x = static_cast<int>(std::ceil(static_cast<float>(parent.urx - parent.ulx) / 2));
    const int half_y = static_cast<int>(std::ceil(static_cast<float>(parent.bry - parent.uly) / 2));
    const int mx = parent.ulx + half_x, my = parent.uly + half_y;
    int cnt[4] = {0, 0, 0, 0};
    int* keys = perm.data() + parent.begin;
    for (int i = 0; i < parent.count; ++i) {
      const int k = keys[i];
      const int q = static_cast<int>(!(xs[k] < mx)) + 2 * static_cast<int>(!(ys[k] < my));  // UL, UR, BL, BR; branch-free
      quad[i] = static_cast<uint8_t>(q);
      ++cnt[q];
    }
    int off[4] = {0, cnt[0], cnt[0] + cnt[1], cnt[0] + cnt[1] + cnt[2]};
    const int start[4] = {off[0], off[1], off[2], off[3]};
    for (int i = 0; i < parent.count; ++i) scratch[off[quad[i]]++] = keys[i];
    std::copy(scratch.begin(), scratch.begin() + parent.count, keys);
    const int bx[4][4] = {{parent.ulx, parent.uly, mx, my}, {mx, parent.uly, parent.urx, my},
                          {parent.ulx, my, mx, parent.bry}, {mx, my, parent.urx, parent.bry}};
    for (int q = 0; q < 4; ++q) {
      if (!cnt[q]) continue;  // empty children never enter the list
      const int c = L.make();
      QNode& nd = L.arena[c];
      nd.ulx = bx[q][0]; nd.uly = bx[q][1]; nd.urx = bx[q][2]; nd.bry = bx[q][3];
      nd.begin = parent.begin + start[q];
      nd.count = cnt[q];
      nd.no_more = cnt[q] == 1;
      L.push_front(c);
      if (cnt[q] > 1) {
        ++n_expand;
        nd.seq = ++seq;
        pending.push_back(c);
      }
    }
  };
  bool finish = false;
  while (!finish) {
    const int prev_size = L.size;
    int n_expand = 0;
    pending.clear();
    for (int i = L.head; i >= 0;) {
      if (L.arena[i].no_more) { i = L.arena[i].next; continue; }
      split(i, n_expand);
      i = L.erase(i);
    }
    if (L.size >= n_target || L.size == prev_size) {
      finish = true;
    } else if (L.size + n_expand * 3 > n_target) {
      while (!finish) {
        const int prev = L.size;
        round = pending;
        pending.clear();
        // std::sort on (size, ExtractorNode*) in the reference (:671-676); ties by creation order here
        std::sort(round.begin(), round.end(), [&](int a, int b) {
          const int sa = L.arena[a].count, sb = L.arena[b].count;
          return sa != sb ? sa < sb : L.arena[a].seq < L.arena[b].seq;
        });
        for (int j = static_cast<int>(round.size()) - 1; j >= 0; --j) {
          int dummy = 0;
          split(round[j], dummy);
          L.erase(round[j]);
          if (L.size >= n_target) break;
        }
        if (L.size >= n_target || L.size == prev) finish = true;
      }
    }
  }
  result.reserve(L.size);
  for (int i = L.head; i >= 0; i = L.arena[i].next) {
    const int* keys = perm.data() + L.arena[i].begin;
    int best = keys[0];
    for (int k = 1; k < L.arena[i].count; ++k)
      if (resp[keys[k]] > resp[best]) best = keys[k];
    result.push_back(best);
  }
  return result;
}

// ---------------------------------------------------------------- Orb
// A handful of helper threads that sleep between calls; run() hands every thread (and the caller) a share.
struct Orb::TreePool {
  std::vector<std::thread> threads;
  std::mutex m;
  std::condition_variable cv, done_cv;
  std::function<void(int)> job;  // argument: worker index 1..threads.size() (the caller is worker 0)
  unsigned generation = 0;
  int pending = 0;
  bool stop = false;
  explicit TreePool(int helpers) {
    for (int i = 0; i < helpers; ++i)
      threads.emplace_back([this, i] {
        unsigned seen = 0;
        for (;;) {
          std::function<void(int)> fn;
          {
            std::unique_lock<std::mutex> lk(m);
            cv.wait(lk, [&] { return stop || generation != seen; });
            if (stop) return;
            seen = generation;
            fn = job;
          }
          fn(i + 1);
          {
            std::lock_guard<std::mutex> lk(m);
            if (--pending == 0) done_cv.notify_one();
          }
        }
      });
  }
  ~TreePool() {
    {
      std::lock_guard<std::mutex> lk(m);
      stop = true;
    }
    cv.notify_all();
    for (auto& t : threads) t.join();
  }
  void run(const std::function<void(int)>& fn) {
    {
      std::lock_guard<std::mutex> lk(m);
      job = fn;
      pending = static_cast<int>(threads.size());
      ++generation;
    }
    cv.notify_all();
    fn(0);
    std::unique_lock<std::mutex> lk(m);
    done_cv.wait(lk, [&] { return pending == 0; });
  }
};

namespace {
std::once_flag g_pattern_once[64];
int cv_round_f(float v) { return static_cast<int>(std::nearbyint(v)); }
}  // namespace

Orb::Orb(int nfeatures, float scale_factor, int nlevels, int ini_th, int min_th, int device)
    : nfeatures_(nfeatures), nlevels_(nlevels), ini_th_(ini_th), min_th_(min_th), device_(device), scale_factor_(scale_factor) {
  if (nfeatures <= 0 || nlevels <= 0 || nlevels > kOrbMaxLevels || !(scale_factor > 1.f) || ini_th <= 0 || min_th <= 0 ||
      ini_th > 255 || min_th > 255)
    fail(SIVO_EINVAL, "ORBextractor: bad parameters (nfeatures %d, scale %.3f, levels %d, th %d/%d)", nfeatures, scale_factor,
         nlevels, ini_th, min_th);
  tab_ = orb_make_tables(nfeatures, scale_factor, nlevels);
  {
    int helpers = std::min(3, nlevels - 1);
    if (const char* e = std::getenv("SIVO_B200_ORB_TREE_THREADS")) helpers = std::max(0, std::min(7, atoi(e) - 1));
    if (helpers > 0) pool_ = std::make_shared<TreePool>(helpers);
  }
  SIVO_CUDA(cudaSetDevice(device_));
  std::call_once(g_pattern_once[device_ & 63], [] { orb_upload_pattern(); });
  {
    // the extractor's kernels are tiny and its caller waits on them twice per image; give them the highest priority so
    // they slot in ahead of the next wave of a long convolution kernel running on the same GPU
    int lo = 0, hi = 0;
    SIVO_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));
    SIVO_CUDA(cudaStreamCreateWithPriority(&stream_, cudaStreamNonBlocking, hi));
  }
  for (auto& e : ev_) SIVO_CUDA(cudaEventCreate(&e));
  SIVO_CUDA(cudaEventCreateWithFlags(&ev_pyr_, cudaEventDisableTiming));
  d_umax_.alloc(sizeof(tab_.umax));
  SIVO_CUDA(cudaMemcpy(d_umax_.p, tab_.umax, sizeof(tab_.umax), cudaMemcpyHostToDevice));
  sel_cap_ = nfeatures + 4 * nlevels + 64;
  // one level of the selection holds up to kTreeSelCap keypoints from the device tree and, short of the capacity error, up to
  // capacity() from the host tree
  d_sel_packed_.alloc(static_cast<size_t>(nlevels) * std::max(kTreeSelCap, sel_cap_) * sizeof(uint32_t));
  d_level_count_.alloc(kOrbMaxLevels * sizeof(int));
  h_sel_packed_.ensure((kOrbMaxLevels + static_cast<size_t>(nlevels) * sel_cap_) * sizeof(uint32_t));
  d_n_err_.alloc(2 * sizeof(int));
  h_n_err_.ensure(2 * sizeof(int));
  d_kps_.alloc(static_cast<size_t>(sel_cap_) * sizeof(sivo_keypoint));
  h_kps_.ensure(static_cast<size_t>(sel_cap_) * sizeof(sivo_keypoint));
  d_desc_.alloc(static_cast<size_t>(sel_cap_) * 32);
  h_desc_.ensure(static_cast<size_t>(sel_cap_) * 32);
  {
    std::vector<float> sc(tab_.scale);
    sc.insert(sc.end(), tab_.inv_scale.begin(), tab_.inv_scale.end());
    d_scales_.alloc(sc.size() * sizeof(float));
    SIVO_CUDA(cudaMemcpy(d_scales_.p, sc.data(), sc.size() * sizeof(float), cudaMemcpyHostToDevice));
  }
  {
    // device quad tree (orb_tree.cu): default; the host tree remains for inputs beyond its shared-memory caps and as the
    // cross-check in the tests (SIVO_B200_ORB_DEVICE_TREE=0 forces it)
    const char* e = std::getenv("SIVO_B200_ORB_DEVICE_TREE");
    device_tree_ = !(e && e[0] == '0');
    for (int l = 0; l < nlevels; ++l) if (tab_.per_level[l] + 8 > kTreeSelCap) device_tree_ = false;
    if (device_tree_) orb_tree_configure();
  }
  d_level_off_.alloc((kOrbMaxLevels + 1) * sizeof(int));
  h_level_off_.ensure((kOrbMaxLevels + 1) * sizeof(int));
}

Orb::~Orb() {
  cudaSetDevice(device_);
  for (auto& e : ev_) if (e) cudaEventDestroy(e);
  if (ev_wait_) cudaEventDestroy(ev_wait_);
  if (ev_pyr_) cudaEventDestroy(ev_pyr_);
  if (copy_stream_) cudaStreamDestroy(copy_stream_);
  if (ev_wait2_) cudaEventDestroy(ev_wait2_);
  if (stream_) cudaStreamDestroy(stream_);
}

void Orb::level_size(int rows, int cols, int level, int* w, int* h) const {
  if (level < 0 || level >= nlevels_) fail(SIVO_EINVAL, "level %d out of range", level);
  // ComputePyramid (:1086-1089)
  float s = tab_.inv_scale[level];
  if (w) *w = cv_round_f(static_cast<float>(cols) * s);
  if (h) *h = cv_round_f(static_cast<float>(rows) * s);
}

void Orb::ensure(int rows, int cols) {
  if (rows == rows_ && cols == cols_) return;
  rows_ = cols_ = 0;  // until the tables below are complete: a refused size must not leave them half rebuilt under the old one
  lt_.nlevels = nlevels_;
  cells_.clear();
  size_t img_off = 0, flat_off = 0;
  for (int l = 0; l < nlevels_; ++l) {
    OrbLevel& lv = lt_.lv[l];
    level_size(rows, cols, l, &lv.w, &lv.h);
    if (lv.w < 2 * kEdge + 7 || lv.h < 2 * kEdge + 7)
      fail(SIVO_EINVAL, "image %dx%d is too small for %d pyramid levels", cols, rows, nlevels_);
    // FAST candidates are packed x:12 | y:12 | response:8 (k_cells): larger levels would wrap silently
    if (lv.w + 2 * kEdge > 4096 || lv.h + 2 * kEdge > 4096)
      fail(SIVO_EINVAL, "image %dx%d exceeds the extractor's 4096-pixel candidate packing", cols, rows);
    lv.pitch = (lv.w + 2 * kEdge + 15) / 16 * 16;
    lv.img_off = img_off;
    lv.flat_off = flat_off;
    img_off += static_cast<size_t>(lv.pitch) * (lv.h + 2 * kEdge);
    img_off = (img_off + 255) / 256 * 256;
    flat_off += static_cast<size_t>(lv.w) * lv.h;
    flat_off = (flat_off + 255) / 256 * 256;
    // cell grid of ComputeKeyPointsOctTree (:759-791)
    const int min_bx = kEdge - 3, min_by = kEdge - 3, max_bx = lv.w - kEdge + 3, max_by = lv.h - kEdge + 3;
    {  // DistributeOctTree's geometry for this level (:547-551), as orb_distribute derives it
      int n_ini = static_cast<int>(std::round(static_cast<float>(max_bx - min_bx) / (max_by - min_by)));
      if (n_ini < 1) n_ini = 1;
      tree_prm_.n_target[l] = tab_.per_level[l];
      tree_prm_.n_ini[l] = n_ini;
      tree_prm_.height[l] = max_by - min_by;
      tree_prm_.hx[l] = static_cast<float>(max_bx - min_bx) / n_ini;
      tree_prm_.scale[l] = tab_.scale[l];
      tree_prm_.size[l] = static_cast<float>(static_cast<int>(31 * tab_.scale[l]));
      tree_prm_.min_b = kEdge - 3;
    }
    const float width = static_cast<float>(max_bx - min_bx), height = static_cast<float>(max_by - min_by);
    const int n_cols = static_cast<int>(width / 30.f), n_rows = static_cast<int>(height / 30.f);
    lv.cell_begin = static_cast<int>(cells_.size());
    // a FAST region under 30 px has no cells (the reference's loops run zero times; its wCell / hCell, ceil(x / 0), are never used)
    const int w_cell = n_cols ? static_cast<int>(std::ceil(width / n_cols)) : 0;
    const int h_cell = n_rows ? static_cast<int>(std::ceil(height / n_rows)) : 0;
    for (int i = 0; i < n_rows && n_cols; ++i) {
      const int ini_y = min_by + i * h_cell;
      int max_y = ini_y + h_cell + 6;
      if (ini_y >= max_by - 3) continue;
      if (max_y > max_by) max_y = max_by;
      for (int j = 0; j < n_cols; ++j) {
        const int ini_x = min_bx + j * w_cell;
        int max_x = ini_x + w_cell + 6;
        if (ini_x >= max_bx - 6) continue;
        if (max_x > max_bx) max_x = max_bx;
        OrbCell c;
        c.level = l;
        c.x0 = static_cast<short>(ini_x); c.y0 = static_cast<short>(ini_y);
        c.x1 = static_cast<short>(max_x); c.y1 = static_cast<short>(max_y);
        cells_.push_back(c);
      }
    }
    lv.cell_end = static_cast<int>(cells_.size());
  }
  pyr_bytes_ = img_off;
  flat_bytes_ = flat_off;
  for (int l = 0; l < nlevels_; ++l) { tree_prm_.cell_begin[l] = lt_.lv[l].cell_begin; tree_prm_.cell_end[l] = lt_.lv[l].cell_end; }
  const int ncells = static_cast<int>(cells_.size());
  d_gray_.alloc(static_cast<size_t>(rows) * cols);
  h_gray_.ensure(static_cast<size_t>(rows) * cols);
  d_pyr_.alloc(pyr_bytes_);
  h_pyr_.ensure(pyr_bytes_);
  d_blur_.alloc(flat_bytes_);
  d_cells_.alloc(std::max<size_t>(1, ncells) * sizeof(OrbCell));
  if (ncells) SIVO_CUDA(cudaMemcpy(d_cells_.p, cells_.data(), ncells * sizeof(OrbCell), cudaMemcpyHostToDevice));
  d_cell_count_.alloc(std::max<size_t>(1, ncells) * sizeof(int));
  d_cell_offset_.alloc((static_cast<size_t>(ncells) + 1) * sizeof(int));
  d_cell_items_.alloc(std::max<size_t>(1, ncells) * kCellCap * sizeof(uint32_t));
  // the compacted candidates are the cell lists back to back, so they never outgrow them; run_host_tree copies only the words a
  // call produced
  cand_cap_ = std::max(1, ncells) * kCellCap;
  d_cand_.alloc(static_cast<size_t>(cand_cap_) * sizeof(uint32_t));
  h_cand_.ensure(static_cast<size_t>(cand_cap_) * sizeof(uint32_t));
  rows_ = rows;
  cols_ = cols;
}

void Orb::run(const uint8_t* gray, int rows, int cols, size_t stride, sivo_keypoint* kps, int cap, int* n, uint8_t* desc,
              uint8_t* const* pyr_out, const size_t* pyr_strides, bool gray_on_device) {
  if (n) *n = 0;
  if (!gray || rows <= 0 || cols <= 0) return;  // `if (_image.empty()) return;` (:1023-1024)
  if (stride < static_cast<size_t>(cols)) fail(SIVO_EINVAL, "ORBextractor: stride smaller than a row");
  const auto w0 = std::chrono::steady_clock::now();
  SIVO_CUDA(cudaSetDevice(device_));
  ensure(rows, cols);
  cudaStream_t s = stream_;
  const uint8_t* src = gray;
  size_t src_pitch = stride;
  if (!gray_on_device && is_pinned_host(gray)) {  // page-locked caller image: no staging copy
    SIVO_CUDA(cudaEventRecord(ev_[0], s));
    SIVO_CUDA(cudaMemcpy2DAsync(d_gray_.p, cols, gray, stride, cols, rows, cudaMemcpyHostToDevice, s));
    src = d_gray_.as<uint8_t>();
    src_pitch = cols;
  } else if (!gray_on_device) {
    uint8_t* hg = h_gray_.as<uint8_t>();
    for (int y = 0; y < rows; ++y) memcpy(hg + static_cast<size_t>(y) * cols, gray + static_cast<size_t>(y) * stride, cols);
    SIVO_CUDA(cudaEventRecord(ev_[0], s));
    SIVO_CUDA(cudaMemcpyAsync(d_gray_.p, hg, static_cast<size_t>(rows) * cols, cudaMemcpyHostToDevice, s));
    src = d_gray_.as<uint8_t>();
    src_pitch = cols;
  } else {
    SIVO_CUDA(cudaEventRecord(ev_[0], s));
  }
  enqueue_front(src, src_pitch, s);
  // the 1.6 MB pyramid read-back (the public mvImagePyramid) leaves on a second stream as soon as the level images exist, under
  // FAST, the quad tree and describe
  bool pyr_direct = pyr_out != nullptr;
  if (pyr_out) {
    for (int l = 0; l < nlevels_; ++l) pyr_direct = pyr_direct && pyr_out[l] && is_pinned_host(pyr_out[l]);
    if (!copy_stream_) SIVO_CUDA(cudaStreamCreateWithFlags(&copy_stream_, cudaStreamNonBlocking));
    SIVO_CUDA(cudaStreamWaitEvent(copy_stream_, ev_pyr_, 0));
    if (pyr_direct) {  // page-locked level buffers (mvImagePyramid storage): strided copies straight into them
      for (int l = 0; l < nlevels_; ++l) {
        const OrbLevel& lv = lt_.lv[l];
        const size_t dst_stride = pyr_strides ? pyr_strides[l] : static_cast<size_t>(lv.w + 2 * kEdge);
        if (dst_stride < static_cast<size_t>(lv.w + 2 * kEdge)) fail(SIVO_EINVAL, "pyramid stride %zu too small for level %d", dst_stride, l);
        SIVO_CUDA(cudaMemcpy2DAsync(pyr_out[l], dst_stride, d_pyr_.as<uint8_t>() + lv.img_off, lv.pitch, lv.w + 2 * kEdge,
                                    lv.h + 2 * kEdge, cudaMemcpyDeviceToHost, copy_stream_));
      }
    } else {
      SIVO_CUDA(cudaMemcpyAsync(h_pyr_.p, d_pyr_.p, pyr_bytes_, cudaMemcpyDeviceToHost, copy_stream_));
    }
  }
  const int* n_err = h_n_err_.as<int>();
  bool host_tree = !device_tree_;
  launches = nlevels_ + 1;  // the pyramid levels and k_cells
  if (device_tree_) {
    // ---- device quad tree: one asynchronous chain, one synchronisation at the end
    SIVO_CUDA(cudaEventRecord(ev_[1], s));
    enqueue_tree_and_describe(d_kps_.as<sivo_keypoint>(), d_desc_.as<uint8_t>(), nullptr, s);
    enqueue_results_readback(s);
    launches += 3;  // blur, distribute, describe
    SIVO_CUDA(cudaStreamSynchronize(s));
    // bits 0-15: a level exceeded the device tree's caps, so the host tree takes the call (the candidates are still on the device)
    host_tree = (n_err[1] & 0xFFFF) != 0;
    if (!host_tree) {
      float a = 0, b2 = 0;
      SIVO_CUDA(cudaEventElapsedTime(&a, ev_[0], ev_[1]));
      SIVO_CUDA(cudaEventElapsedTime(&b2, ev_[1], ev_[3]));
      device_ms = a + b2;
      tree_ms = 0.f;
      last_off_.clear();  // candidates() fetches them from the device on demand
    }
  }
  if (host_tree) run_host_tree(w0);
  if (pyr_out) SIVO_CUDA(cudaStreamSynchronize(copy_stream_));
  if (n_err[1] & (1 << 30)) fail(SIVO_ERANGE, "ORBextractor: more keypoints than the workspace holds (%d)", sel_cap_);
  const int total = n_err[0];
  if (n) *n = total;
  if (total > cap) fail(SIVO_ERANGE, "ORBextractor: %d keypoints but the caller's buffers hold %d", total, cap);
  if (kps && total) memcpy(kps, h_kps_.p, static_cast<size_t>(total) * sizeof(sivo_keypoint));
  if (desc && total) memcpy(desc, h_desc_.p, static_cast<size_t>(total) * 32);
  if (pyr_out && !pyr_direct) {
    for (int l = 0; l < nlevels_; ++l) {
      if (!pyr_out[l]) continue;
      const OrbLevel& lv = lt_.lv[l];
      const size_t dst_stride = pyr_strides ? pyr_strides[l] : static_cast<size_t>(lv.w + 2 * kEdge);
      if (dst_stride < static_cast<size_t>(lv.w + 2 * kEdge)) fail(SIVO_EINVAL, "pyramid stride %zu too small for level %d", dst_stride, l);
      const uint8_t* srcl = h_pyr_.as<uint8_t>() + lv.img_off;
      for (int y = 0; y < lv.h + 2 * kEdge; ++y)
        memcpy(pyr_out[l] + static_cast<size_t>(y) * dst_stride, srcl + static_cast<size_t>(y) * lv.pitch, lv.w + 2 * kEdge);
    }
  }
}

// ---- host quad tree: candidates down, orb_distribute per level on the pool, the selection up, the describe pass
void Orb::run_host_tree(std::chrono::steady_clock::time_point w0) {
  cudaStream_t s = stream_;
  enqueue_compact(s);
  // the level offsets first: the candidates' copy then moves the words this call produced, not the whole workspace
  SIVO_CUDA(cudaMemcpyAsync(h_level_off_.p, d_level_off_.p, (nlevels_ + 1) * sizeof(int), cudaMemcpyDeviceToHost, s));
  SIVO_CUDA(cudaStreamSynchronize(s));
  const int* loff = h_level_off_.as<int>();
  SIVO_CUDA(cudaMemcpyAsync(h_cand_.p, d_cand_.p, static_cast<size_t>(loff[nlevels_]) * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  SIVO_CUDA(cudaEventRecord(ev_[1], s));
  // the blur overlaps the host quad tree (the device tree's chain, if it ran, has blurred already)
  if (!device_tree_) orb_launch_blur(d_pyr_.as<uint8_t>(), d_blur_.as<uint8_t>(), lt_, s);
  launches += device_tree_ ? 3 : 4;  // compact's two, describe, and the blur if it has not run
  static const bool trace = [] { const char* e = std::getenv("SIVO_B200_ORB_TRACE"); return e && e[0] == '1'; }();
  const auto w1 = std::chrono::steady_clock::now();
  SIVO_CUDA(cudaEventSynchronize(ev_[1]));
  const auto w2 = std::chrono::steady_clock::now();

  const uint32_t* cand = h_cand_.as<uint32_t>();
  auto t0 = std::chrono::steady_clock::now();
  last_off_.assign(loff, loff + nlevels_ + 1);
  last_cand_.assign(cand, cand + loff[nlevels_]);
  const int min_b = kEdge - 3;
  auto tree_level = [&](int l) {
    const OrbLevel& lv = lt_.lv[l];
    const int b = loff[l], m = loff[l + 1] - b;
    std::vector<float>&xs = lxs_[l], &ys = lys_[l], &rs = lrs_[l];
    xs.resize(m); ys.resize(m); rs.resize(m);
    for (int i = 0; i < m; ++i) {
      const uint32_t c = cand[b + i];
      xs[i] = static_cast<float>(c & 0xFFF);
      ys[i] = static_cast<float>((c >> 12) & 0xFFF);
      rs[i] = static_cast<float>(c >> 24);
    }
    lkeep_[l] = orb_distribute(xs.data(), ys.data(), rs.data(), m, min_b, lv.w - kEdge + 3, min_b, lv.h - kEdge + 3, tab_.per_level[l]);
  };
  {
    // longest-processing-time assignment of the levels to the caller + helpers
    const int workers = pool_ ? static_cast<int>(pool_->threads.size()) + 1 : 1;
    int order[kOrbMaxLevels], owner[kOrbMaxLevels], load[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int l = 0; l < nlevels_; ++l) order[l] = l;
    std::sort(order, order + nlevels_, [&](int a, int b) { return loff[a + 1] - loff[a] > loff[b + 1] - loff[b]; });
    for (int i = 0; i < nlevels_; ++i) {
      int w = 0;
      for (int k = 1; k < workers; ++k) if (load[k] < load[w]) w = k;
      owner[order[i]] = w;
      load[w] += loff[order[i] + 1] - loff[order[i]] + 64;
    }
    std::string worker_error;
    std::mutex err_m;
    auto share = [&](int w) {
      try {
        for (int l = 0; l < nlevels_; ++l) if (owner[l] == w) tree_level(l);
      } catch (const std::exception& e) {
        std::lock_guard<std::mutex> lk(err_m);
        worker_error = e.what();
      }
    };
    if (pool_) pool_->run(share); else share(0);
    if (!worker_error.empty()) fail(SIVO_EINVAL, "ORBextractor: quad tree failed: %s", worker_error.c_str());
  }
  // the selection in the device tree's form: kept index k of level l is candidate loff[l] + k, whose packed word is the entry;
  // a level longer than capacity() means more keypoints than that in all, which k_describe reports without reading the words
  int stride = 0;
  for (int l = 0; l < nlevels_; ++l) stride = std::max(stride, static_cast<int>(lkeep_[l].size()));
  stride = std::min(stride, sel_cap_);
  int* count = h_sel_packed_.as<int>();
  uint32_t* sel = h_sel_packed_.as<uint32_t>() + kOrbMaxLevels;
  for (int l = 0; l < nlevels_; ++l) {
    count[l] = static_cast<int>(lkeep_[l].size());
    for (int k = 0; k < std::min(count[l], stride); ++k) sel[l * stride + k] = cand[loff[l] + lkeep_[l][k]];
  }
  tree_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
  SIVO_CUDA(cudaEventRecord(ev_[2], s));
  SIVO_CUDA(cudaMemcpyAsync(d_level_count_.p, count, nlevels_ * sizeof(int), cudaMemcpyHostToDevice, s));
  SIVO_CUDA(cudaMemcpyAsync(d_sel_packed_.p, sel, static_cast<size_t>(nlevels_) * stride * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
  SIVO_CUDA(cudaMemsetAsync(d_n_err_.p, 0, 2 * sizeof(int), s));
  enqueue_describe(stride, d_kps_.as<sivo_keypoint>(), d_desc_.as<uint8_t>(), nullptr, s);
  enqueue_results_readback(s);
  const auto w3 = std::chrono::steady_clock::now();
  SIVO_CUDA(cudaStreamSynchronize(s));
  if (trace) {
    auto ms = [](auto a, auto b) { return std::chrono::duration<float, std::milli>(b - a).count(); };
    fprintf(stderr, "[orb %p] enqueue %.3f wait1 %.3f tree %.3f enqueue2 %.3f wait2 %.3f ms, %d candidates\n", static_cast<void*>(this),
            ms(w0, w1), ms(w1, w2), tree_ms, ms(t0, w3) - tree_ms, ms(w3, std::chrono::steady_clock::now()), loff[nlevels_]);
  }
  float a = 0, b2 = 0;
  SIVO_CUDA(cudaEventElapsedTime(&a, ev_[0], ev_[1]));
  SIVO_CUDA(cudaEventElapsedTime(&b2, ev_[2], ev_[3]));
  device_ms = a + b2;
}

void Orb::enqueue_front(const uint8_t* src, size_t src_pitch, cudaStream_t s) {
  const int ncells = static_cast<int>(cells_.size());
  orb_launch_pyramid(src, rows_, cols_, src_pitch, d_pyr_.as<uint8_t>(), lt_, s);
  SIVO_CUDA(cudaEventRecord(ev_pyr_, s));  // the level images are final: their read-back can start on the copy stream
  orb_launch_cells(d_pyr_.as<uint8_t>(), lt_, d_cells_.as<OrbCell>(), ncells, ini_th_, min_th_, d_cell_count_.as<int>(),
                   d_cell_items_.as<uint32_t>(), s);
  compacted_ = false;  // the device tree reads the cell lists directly; the host path and the test hook compact on demand
}

void Orb::enqueue_compact(cudaStream_t s) {
  if (compacted_) return;
  orb_launch_compact(lt_, d_cells_.as<OrbCell>(), static_cast<int>(cells_.size()), d_cell_count_.as<int>(), d_cell_items_.as<uint32_t>(),
                     d_cell_offset_.as<int>(), d_level_off_.as<int>(), d_cand_.as<uint32_t>(), cand_cap_, s);
  compacted_ = true;
}

void Orb::enqueue_tree_and_describe(sivo_keypoint* kps_dev, uint8_t* desc_dev, long long* count_dev, cudaStream_t s) {
  int* n_dev = d_n_err_.as<int>();
  SIVO_CUDA(cudaMemsetAsync(n_dev, 0, 2 * sizeof(int), s));
  orb_launch_blur(d_pyr_.as<uint8_t>(), d_blur_.as<uint8_t>(), lt_, s);
  orb_launch_distribute(nullptr, nullptr, d_cell_items_.as<uint32_t>(), d_cell_count_.as<int>(), tree_prm_, nlevels_,
                        d_sel_packed_.as<uint32_t>(), d_level_count_.as<int>(), n_dev + 1, s);
  enqueue_describe(kTreeSelCap, kps_dev, desc_dev, count_dev, s);
}

void Orb::enqueue_describe(int stride, sivo_keypoint* kps_dev, uint8_t* desc_dev, long long* count_dev, cudaStream_t s) {
  int* n_dev = d_n_err_.as<int>();
  orb_launch_describe_dev(d_pyr_.as<uint8_t>(), d_blur_.as<uint8_t>(), lt_, d_sel_packed_.as<uint32_t>(), d_level_count_.as<int>(), stride,
                          tree_prm_, sel_cap_, d_umax_.as<int>(), kps_dev, desc_dev, n_dev, count_dev, n_dev + 1, s);
}

void Orb::enqueue_results_readback(cudaStream_t s) {
  SIVO_CUDA(cudaMemcpyAsync(h_n_err_.p, d_n_err_.p, 2 * sizeof(int), cudaMemcpyDeviceToHost, s));
  SIVO_CUDA(cudaMemcpyAsync(h_kps_.p, d_kps_.p, static_cast<size_t>(sel_cap_) * sizeof(sivo_keypoint), cudaMemcpyDeviceToHost, s));
  SIVO_CUDA(cudaMemcpyAsync(h_desc_.p, d_desc_.p, static_cast<size_t>(sel_cap_) * 32, cudaMemcpyDeviceToHost, s));
  SIVO_CUDA(cudaEventRecord(ev_[3], s));
}

void Orb::enqueue_device(const uint8_t* gray_dev, int rows, int cols, size_t pitch, sivo_keypoint* kps_dev, uint8_t* desc_dev,
                         long long* count_dev) {
  if (!device_tree_) fail(SIVO_EINVAL, "ORBextractor: the asynchronous form needs the device quad tree");
  if (!gray_dev || !kps_dev || !desc_dev || rows <= 0 || cols <= 0 || pitch < static_cast<size_t>(cols))
    fail(SIVO_EINVAL, "ORBextractor: bad arguments");
  SIVO_CUDA(cudaSetDevice(device_));
  ensure(rows, cols);
  enqueue_front(gray_dev, pitch, stream_);
  enqueue_tree_and_describe(kps_dev, desc_dev, count_dev, stream_);
  launches = nlevels_ + 4;
  last_off_.clear();
}

void Orb::stream_wait(cudaStream_t consumer) {
  if (!ev_wait_) SIVO_CUDA(cudaEventCreateWithFlags(&ev_wait_, cudaEventDisableTiming));
  SIVO_CUDA(cudaSetDevice(device_));
  SIVO_CUDA(cudaEventRecord(ev_wait_, stream_));
  SIVO_CUDA(cudaStreamWaitEvent(consumer, ev_wait_, 0));
}

void Orb::wait_for_stream(cudaStream_t producer) {
  SIVO_CUDA(cudaSetDevice(device_));
  if (!ev_wait2_) SIVO_CUDA(cudaEventCreateWithFlags(&ev_wait2_, cudaEventDisableTiming));
  SIVO_CUDA(cudaEventRecord(ev_wait2_, producer));
  SIVO_CUDA(cudaStreamWaitEvent(stream_, ev_wait2_, 0));
}

void Orb::wait_event(cudaEvent_t e) {
  SIVO_CUDA(cudaSetDevice(device_));
  SIVO_CUDA(cudaStreamWaitEvent(stream_, e, 0));
}

int Orb::device_tree_status() {
  if (!device_tree_) return 0;
  SIVO_CUDA(cudaSetDevice(device_));
  int v[2] = {0, 0};
  SIVO_CUDA(cudaMemcpyAsync(v, d_n_err_.p, sizeof v, cudaMemcpyDeviceToHost, stream_));
  SIVO_CUDA(cudaStreamSynchronize(stream_));
  return v[1];
}

void Orb::candidates(int level, int* xs, int* ys, int* resp, int cap, int* n) const {
  if (last_off_.empty() && rows_ > 0) {  // device-tree runs leave the candidates on the device: fetch them on demand
    SIVO_CUDA(cudaSetDevice(device_));
    const_cast<Orb*>(this)->enqueue_compact(stream_);
    last_off_.resize(nlevels_ + 1);
    SIVO_CUDA(cudaMemcpyAsync(last_off_.data(), d_level_off_.p, (nlevels_ + 1) * sizeof(int), cudaMemcpyDeviceToHost, stream_));
    SIVO_CUDA(cudaStreamSynchronize(stream_));
    const int total = std::min(last_off_[nlevels_], cand_cap_);
    last_cand_.resize(std::max(total, 1));
    SIVO_CUDA(cudaMemcpyAsync(last_cand_.data(), d_cand_.p, static_cast<size_t>(total) * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream_));
    SIVO_CUDA(cudaStreamSynchronize(stream_));
  }
  if (level < 0 || level + 1 >= static_cast<int>(last_off_.size())) fail(SIVO_EINVAL, "no candidates for level %d", level);
  const uint32_t* v = last_cand_.data() + last_off_[level];
  const int m = last_off_[level + 1] - last_off_[level];
  if (n) *n = m;
  if (m > cap) fail(SIVO_ERANGE, "level %d has %d candidates, buffer holds %d", level, m, cap);
  for (int i = 0; i < m; ++i) {
    if (xs) xs[i] = static_cast<int>(v[i] & 0xFFF);
    if (ys) ys[i] = static_cast<int>((v[i] >> 12) & 0xFFF);
    if (resp) resp[i] = static_cast<int>(v[i] >> 24);
  }
}

}  // namespace sivo
