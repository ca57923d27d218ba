// ORB extractor: host twin of `SIVO::ORBextractor` (src/orbslam/ORBextractor.cc) driving the kernels in
// orb_kernels.cu.  One instance = one CUDA stream + its own workspace, so two instances can run
// concurrently from two threads as Frame.cc:126-129 does.
#pragma once
#include <condition_variable>
#include <cstdlib>
#include <functional>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

#include "common.h"

namespace sivo {

constexpr int kOrbMaxLevels = 16;
constexpr int kEdge = 19;        // EDGE_THRESHOLD (ORBextractor.cc:72)
constexpr int kHalfPatch = 15;   // HALF_PATCH_SIZE
constexpr int kCellCap = 1024;   // per-cell candidate slots (3x3 NMS keeps <= 1/4 of a <= 62x62 interior)

struct OrbLevel {
  int w, h;            // level image size
  int pitch;           // bytes per row of the bordered buffer ((w + 38) rounded up to 16)
  size_t img_off;      // offset of the bordered buffer in the pyramid arena
  size_t flat_off;     // offset of the w*h planes (score map, blurred image) in their arenas
  int cell_begin, cell_end;
};

struct OrbCell {
  int level;
  short x0, y0, x1, y1;  // FAST sub-image rectangle in level coordinates (ORBextractor.cc:776-798)
};

struct OrbLevelTable {
  int nlevels;
  OrbLevel lv[kOrbMaxLevels];
};

// device quad tree (orb_tree.cu): shared-memory caps of one level
constexpr int kTreeKeyCap = 8192;   // FAST candidates of one level
constexpr int kTreeNodeCap = 4096;  // nodes ever created for one level
constexpr int kTreeListCap = 2048;  // list length / children of one round
constexpr int kTreeSelCap = 1024;   // retained keypoints of one level (<= n_target + 2)

struct OrbTreeParams {
  int n_target[kOrbMaxLevels];  // mnFeaturesPerLevel
  int n_ini[kOrbMaxLevels];     // initial cells: round(width / height) of the level's FAST region (ORBextractor.cc:551)
  int height[kOrbMaxLevels];    // maxY - minY
  float hx[kOrbMaxLevels];      // width / n_ini
  float scale[kOrbMaxLevels];   // mvScaleFactor
  float size[kOrbMaxLevels];    // float(int(PATCH_SIZE * mvScaleFactor[level]))
  int cell_begin[kOrbMaxLevels], cell_end[kOrbMaxLevels];  // the level's FAST cells in the global cell list
  int min_b;                    // EDGE_THRESHOLD - 3: level coordinate of candidate (0, 0)
};

struct OrbSelected {  // one retained keypoint, level coordinates
  short x, y;
  short level;
  short pad;
};

// Programmatic dependent launch for the extractor's chain of short dependent kernels: every kernel starts with
// `griddepcontrol.launch_dependents; griddepcontrol.wait;` (ORB_PDL_PROLOGUE), so the next grid of the stream is scheduled while
// this one drains and only its launch latency -- not its work -- overlaps (the wait returns once the previous grid has completed
// and flushed).  Opt-in (SIVO_B200_ORB_PDL=1; without the attribute the prologue is a no-op): the early CTAs of the next small
// kernel sit on SMs the convolution CTAs need.
#define ORB_PDL_PROLOGUE() asm volatile("griddepcontrol.launch_dependents;\n\tgriddepcontrol.wait;" ::: "memory")
template <class... KArgs, class... Args>
inline void orb_launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args... args) {
  static const bool pdl = [] { const char* e = std::getenv("SIVO_B200_ORB_PDL"); return e && e[0] == '1'; }();
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  SIVO_CUDA(cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...));
}

// ---- kernels (orb_kernels.cu)
void orb_launch_pyramid(const uint8_t* gray, int rows, int cols, size_t gray_pitch, uint8_t* pyr, const OrbLevelTable& t,
                        cudaStream_t s);
void hamming_best2(int device, const uint8_t* query, int nq, const uint8_t* train, int nt, const int* cand_off, const int* cand_idx,
                   const int* train_level, int* out5);
void orb_launch_score(const uint8_t* pyr, uint8_t* score, const OrbLevelTable& t, int t_min, cudaStream_t s);
// score == nullptr: the cells score their own pixels from `pyr` (no score-map pass)
void orb_launch_cells(const uint8_t* score, const uint8_t* pyr, const OrbLevelTable& t, const OrbCell* cells, int ncells, int ini_th,
                      int min_th, int* cell_count, uint32_t* cell_items, cudaStream_t s);
void orb_launch_compact(const OrbLevelTable& t, const OrbCell* cells, int ncells, const int* cell_count,
                        const uint32_t* cell_items, int* cell_offset, int* level_offsets, uint32_t* cand, int cand_cap,
                        cudaStream_t s);
void orb_launch_blur(const uint8_t* pyr, uint8_t* blur, const OrbLevelTable& t, cudaStream_t s);
void orb_launch_describe(const uint8_t* pyr, const uint8_t* blur, const OrbLevelTable& t, const OrbSelected* sel, int n,
                         const int* umax, float* angles, uint8_t* desc, cudaStream_t s);
// the same for a keypoint count that lives on the device (<= cap): angles go straight into the keypoint records
// Device-tree form: per-level selections (sel_packed[l * kTreeSelCap + i], level_count[l]) -> level-major keypoint records
// (ComputeKeyPointsOctTree :824-835 + the final scaling of operator() :1071-1078, angle from IC_Angle) and descriptors;
// *n_out (and *n_out_i64 if given) = the keypoint count, bit 30 of *error if it exceeds cap.
void orb_launch_describe_dev(const uint8_t* pyr, const uint8_t* blur, const OrbLevelTable& t, const uint32_t* sel_packed,
                             const int* level_count, const OrbTreeParams& prm, int cap, const int* umax, sivo_keypoint* kps,
                             uint8_t* desc, int* n_out, long long* n_out_i64, int* error, cudaStream_t s);
// DistributeOctTree on the device, one block per level (orb_tree.cu), then the level-major keypoint records
void orb_launch_distribute(const uint32_t* cand, const int* level_off, const uint32_t* cell_items, const int* cell_count,
                           const OrbTreeParams& prm, int nlevels, uint32_t* sel_packed, int* level_count, int* error, cudaStream_t s);
void orb_tree_configure();  // raises k_distribute's dynamic shared-memory limit on the current device
void orb_upload_pattern();  // copies the rBRIEF pair table into constant memory (once per device)

// ---- host (orb_host.cu)
struct OrbTables {
  std::vector<float> scale, inv_scale, sigma2, inv_sigma2;
  std::vector<int> per_level;
  int umax[kHalfPatch + 1];
};
OrbTables orb_make_tables(int nfeatures, float scale_factor, int nlevels);

// DistributeOctTree (ORBextractor.cc:544-750) with the documented tie rule; returns kept indices in
// the reference's output order.
std::vector<int> orb_distribute(const float* xs, const float* ys, const float* resp, int n, int min_x, int max_x, int min_y,
                                int max_y, int n_target);

class Orb {
 public:
  Orb(int nfeatures, float scale_factor, int nlevels, int ini_th, int min_th, int device);
  ~Orb();
  void run(const uint8_t* gray, int rows, int cols, size_t stride, sivo_keypoint* kps, int cap, int* n, uint8_t* desc,
           uint8_t* const* pyr_out, const size_t* pyr_strides, bool gray_on_device = false);
  void level_size(int rows, int cols, int level, int* w, int* h) const;
  const OrbTables& tables() const { return tab_; }
  // device-resident state of the last run, for the stereo stage (no host round trip of the pyramids)
  const uint8_t* dev_pyramid() const { return d_pyr_.as<uint8_t>(); }
  const OrbLevelTable& levels() const { return lt_; }
  int device() const { return device_; }
  bool has_run() const { return rows_ > 0; }
  int nlevels() const { return nlevels_; }
  void candidates(int level, int* xs, int* ys, int* resp, int cap, int* n) const;
  // Fully asynchronous form (needs the device quad tree): enqueues the whole extractor on this handle's stream and returns.
  // Results stay on the device: kps_dev (>= capacity() records), desc_dev (capacity() x 32 bytes), *count_dev (int64).
  void enqueue_device(const uint8_t* gray_dev, int rows, int cols, size_t pitch, sivo_keypoint* kps_dev, uint8_t* desc_dev,
                      long long* count_dev);
  // makes `consumer` wait (on the device) for everything enqueued on this handle's stream so far
  void stream_wait(cudaStream_t consumer);
  void wait_for_stream(cudaStream_t producer);
  void wait_event(cudaEvent_t e);
  // bit l set: level l of the last enqueue_device() did not fit the device tree (the results are then not valid)
  int device_tree_status();
  int capacity() const { return sel_cap_; }
  bool device_tree() const { return device_tree_; }
  float device_ms = 0, tree_ms = 0;
  int launches = 0;

 private:
  void ensure(int rows, int cols);
  void enqueue_front(const uint8_t* src, size_t src_pitch, cudaStream_t s);
  void enqueue_compact(cudaStream_t s);
  bool compacted_ = false;
  void enqueue_tree_and_describe(sivo_keypoint* kps_dev, uint8_t* desc_dev, long long* count_dev, cudaStream_t s);
  bool device_tree_ = true;
  OrbTreeParams tree_prm_{};
  DevBuf d_sel_packed_, d_level_count_, d_n_err_, d_kps_;
  PinnedBuf h_n_err_, h_kps_;
  cudaEvent_t ev_wait_ = nullptr, ev_wait2_ = nullptr, ev_pyr_ = nullptr;
  cudaStream_t copy_stream_ = nullptr;
  int nfeatures_, nlevels_, ini_th_, min_th_, device_;
  float scale_factor_;
  OrbTables tab_;
  int rows_ = 0, cols_ = 0;
  OrbLevelTable lt_{};
  std::vector<OrbCell> cells_;
  cudaStream_t stream_ = nullptr;
  cudaEvent_t ev_[4] = {nullptr, nullptr, nullptr, nullptr};
  DevBuf d_gray_, d_pyr_, d_score_, d_blur_, d_cells_, d_cell_count_, d_cell_items_, d_cell_offset_, d_level_off_, d_cand_,
      d_sel_, d_umax_, d_angles_, d_desc_;
  PinnedBuf h_gray_, h_cand_, h_level_off_, h_sel_, h_angles_, h_desc_, h_pyr_;
  size_t pyr_bytes_ = 0, flat_bytes_ = 0;
  int cand_cap_ = 0, sel_cap_ = 0;
  mutable std::vector<uint32_t> last_cand_;  // last call's packed candidates (x | y << 12 | resp << 24), all levels (test hook)
  mutable std::vector<int> last_off_;        // per-level offsets into last_cand_
  // host quad tree: the pyramid levels are independent, so they are distributed over a few persistent helper threads
  // (largest level first); results are assembled in level order, so the output is the sequential one
  struct TreePool;
  std::shared_ptr<TreePool> pool_;
  std::vector<float> lxs_[kOrbMaxLevels], lys_[kOrbMaxLevels], lrs_[kOrbMaxLevels];
  std::vector<int> lkeep_[kOrbMaxLevels];
};

}  // namespace sivo
