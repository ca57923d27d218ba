// Bayesian SegNet executor: prototxt + caffemodel -> a static list of device ops over NHWC tensors.
// Host-side twin of `SIVO::BayesianSegNet` (src/bayesian_segnet/bayesian_segnet.cpp).
#pragma once
#include <cuda_fp16.h>

#include <map>
#include <memory>
#include <string>
#include <vector>

#include "caffemodel.h"
#include "common.h"
#include "prototxt.h"
#include "segnet_kernels.h"

namespace sivo {

struct ConvTcPlan;  // conv_tc.cu

struct Tensor {
  std::string name;
  TensorView v;
  DevBuf buf;
  bool is_mask = false;  // u8 2-bit argmax codes, dims = pooled dims
  bool elided = false;   // a fusion consumes this blob in registers: it is never written (blob() refuses to read it)
  // >= 0: the max-unpool of tensor `derived_from` by mask tensor `derived_mask`, which its consumer expands as it loads: no
  // kernel writes it, and blob() computes it on demand into a buffer allocated on that first read
  int derived_from = -1, derived_mask = -1;
};

struct Op {
  enum Kind { Input, LRN, Pad8, InputPad8, DropoutUnpool, Conv, Pool, Unpool, Dropout, Reduce } kind = Input;
  std::string layer;
  int in = -1, in2 = -1, out = -1, out2 = -1;
  // LRN
  int lrn_size = 5;
  float lrn_alpha = 1.f, lrn_beta = 0.75f, lrn_k = 1.f;
  // Conv
  int k = 0, pad = 0, cin = 0, cout = 0, cin_p = 0, cout_p = 0;
  std::vector<float> h_w_raw;  // the caffemodel's (cout, cin, k, k) floats, unrounded (the composed classifier's input)
  std::vector<float> h_bias, h_bn_scale, h_bn_shift;  // [cout_p] host copies (the tensor-core kernels take them as kernel parameters)
  int fold_kw = 0;  // > 0: KxK conv over 3 channels run as a Kx1 conv over the window-folded padded input (conv_tc.cu)
  bool relu = false, has_bn = false;
  float slope = 0.f;
  DevBuf w_simt, bias, bn_scale, bn_shift;  // the SIMT kernel's weights [tap][cin_p][cout_p] float and constants
  DevBuf w_tc;                              // the tensor-core kernels' weights [tap][cout_p][cin_p] half
  // split-operand fp32 mode (precision fp32 on the tensor-core engine): x = hi + lo and w * 2^s = hi + lo in half, and
  // x * w ~= (x_hi w_hi + x_hi w_lo + x_lo w_hi) * 2^-s accumulated in fp32 -- three MMAs per tap, ~2^-22 relative per product.
  // w_tc holds [tap][cout_p][3 cin_p] = per 64-channel chunk [W_hi | W_lo | W_hi]; a_split the [hi Cin | lo Cin] planes of the input.
  bool split = false;
  float acc_scale = 1.f;
  DevBuf a_split;
  std::shared_ptr<ConvTcPlan> tc;
  bool use_tc = false;
  double flops = 0;       // algorithmic (the reference's operation count), for this op's batch
  double flops_exec = 0;  // what the launch executes: differs for the composed classifier (0.25x) and the split-operand mode (3x)
  // Dropout
  int drop_layer = 0;
  float drop_scale = 2.f;
};

class SegNet {
 public:
  // sample_count 0: the whole frame, samples [0, T).  Otherwise a latency-mode shard owning samples
  // [sample_begin, sample_begin + sample_count) of a frame of T (= opt.T or the prototxt's batch) samples.
  SegNet(const std::string& prototxt, const std::string& caffemodel, const sivo_segnet_options& opt, int sample_begin = 0,
         int sample_count = 0);
  ~SegNet();
  int width() const { return W_; }
  int height() const { return H_; }
  int T() const { return T_; }
  int sample_begin() const { return s0_; }
  int sample_count() const { return ns_; }
  int classes() const { return n_classes_; }
  void set_frame(uint64_t f) { frame_ = f; }
  void run_host(const uint8_t* bgr, int rows, int cols, size_t stride, uint8_t* classes, double* conf, double* ent);
  // segmentImage (run_host) additionally leaves the classes and f32 copies of the two maps at these device addresses, complete
  // when it returns (all NULL: off)
  void set_record_outputs(uint8_t* classes_dev, float* conf32_dev, float* ent32_dev) {
    rec_classes_ = classes_dev; rec_conf32_ = conf32_dev; rec_ent32_ = ent32_dev;
  }
  // conf32 / ent32 (optional): single-precision copies of the two maps, e.g. straight into the packed multi-GPU record
  void run_device(const uint8_t* bgr_dev, uint8_t* classes_dev, double* conf_dev, double* ent_dev, cudaStream_t s, float* conf32_dev = nullptr,
                  float* ent32_dev = nullptr);
  // latency mode: the shard's samples through the net, then sum_dev[H*W][16] (double) = their sum of per-sample softmax
  void run_partial(const uint8_t* bgr_dev, double* sum_dev, cudaStream_t s);
  // the maps from a sum over all T samples of the frame (e.g. the shards' sums reduced over ranks); any output may be NULL
  void finalize(const double* sum_dev, uint8_t* classes_dev, double* conf_dev, double* ent_dev, float* conf32_dev, float* ent32_dev,
                cudaStream_t s);
  // computeVariance over the samples of the last run (the logits feeding the Reduce op): per pixel the sample variance of the
  // probability of class classes[pix] (0 where it is >= the class count).  The device forms run on `s` (NULL = the handle's
  // own stream), which must be ordered after that run and before the next; the host form synchronises.
  void variance_host(const uint8_t* classes, double* variance);
  void variance_device(const uint8_t* classes_dev, double* variance_dev, cudaStream_t s);
  // latency mode: moments_dev[H*W][2] = (sum p, sum p^2) over this shard's samples; the variance from the moments summed over
  // all T samples of the frame
  void variance_partial(const uint8_t* classes_dev, double* moments_dev, cudaStream_t s);
  void variance_finalize(const double* moments_dev, double* variance_dev, cudaStream_t s);
  void semantic_keys(const sivo_keypoint* kps, int n, int max_static_class, uint8_t* kp_class, double* kp_conf, double* kp_entropy,
                     int* keep_idx, int* n_keep);
  // the same on device buffers with a device-resident count (<= cap), on `s` (NULL = the stream of the last run); no host sync
  void semantic_keys_device(const sivo_keypoint* kps_dev, const long long* count_dev, int cap, int max_static_class, uint8_t* kp_class_dev,
                            double* kp_conf_dev, double* kp_entropy_dev, int* keep_idx_dev, long long* n_keep_dev, cudaStream_t s);
  void blob(const std::string& name, float* out, size_t cap, int* n, int* c, int* h, int* w);
  void set_profiling(bool on) { profiling_ = on; }
  float conv_ms = 0, other_ms = 0, reduce_ms = 0, total_ms = 0;
  std::vector<float> op_ms;  // per launch of the last profiled run, in launch order
  size_t n_ops() const { return ops_.size(); }
  const Op& op_at(size_t i) const { return ops_[i]; }
  int launches = 0;
  double flops_dedup = 0, flops_naive = 0;

 private:
  int add_tensor(const std::string& name, int n, int c, int h, int w, int cs, DType dt, bool mask = false);
  void build(const NetSpec& net, const WeightMap& weights);
  void enqueue(const uint8_t* bgr_dev, uint8_t* classes_dev, double* conf_dev, double* ent_dev, cudaStream_t s, bool timed);
  // one frame of the op list (graph replay or plain launches) with the per-frame arguments `fa`, ending as reduce_ says
  void launch_frame(FrameArgs fa, cudaStream_t s);
  void require_whole_frame(const char* what) const;
  // the logits of the last run's samples (the Reduce op's input); fails if the handle has not run yet
  const TensorView& last_logits(const char* what) const;

  sivo_segnet_options opt_;
  // T_: samples of the frame (the mean divides by it); this handle runs samples [s0_, s0_ + ns_) (ns_ = T_ unless a shard)
  int device_ = 0, T_ = 0, H_ = 0, W_ = 0, n_classes_ = 0, s0_ = 0, ns_ = 0;
  DType act_ = DType::F16;
  uint64_t frame_ = 0;
  bool profiling_ = false;
  std::vector<std::unique_ptr<Tensor>> tensors_;
  std::map<std::string, int> by_name_;
  std::vector<Op> ops_;
  cudaStream_t stream_ = nullptr;
  DevBuf d_bgr_, d_classes_, d_conf_, d_ent_, d_frame_;
  PinnedBuf h_in_, h_classes_, h_conf_, h_ent_;
  // where the last run left its maps on the device, and the stream it ran on (semantic_keys reads them)
  const uint8_t* last_classes_ = nullptr;
  const double* last_conf_ = nullptr;
  const double* last_ent_ = nullptr;
  cudaStream_t last_stream_ = nullptr;
  // stream of the last run_device / run_partial; non-NULL once a frame has been issued, so that the logits tensor holds its
  // samples (the variance reads them)
  cudaStream_t run_stream_ = nullptr;
  DevBuf d_var_classes_, d_var_;  // device staging of the host-buffer variance call
  DevBuf d_kp_, d_kp_out_;
  PinnedBuf h_kp_, h_kp_out_;
  std::vector<cudaEvent_t> events_;
  // how the op list's Reduce op runs: the full MC reduction, or the latency-mode partial sum (run_partial)
  enum class ReduceMode { Full, Partial };
  ReduceMode reduce_ = ReduceMode::Full;
  // the op list captured as CUDA graphs (one launch per frame), one per (stream, ReduceMode) the caller has used, most recently
  // used first.  The kernels read the per-frame pointers from FrameArgs, so every buffer set replays the same graph.
  struct GraphEntry { cudaStream_t stream; ReduceMode reduce; cudaGraphExec_t exec; };
  std::vector<GraphEntry> graphs_;
  static constexpr size_t kMaxGraphs = 32;
  bool graph_ok_ = true;
  // device-resident copies run_host leaves for a packed multi-GPU record (set_record_outputs)
  uint8_t* rec_classes_ = nullptr;
  float* rec_conf32_ = nullptr;
  float* rec_ent32_ = nullptr;
};

// Packs convolution `op`'s weights (`w`: the caffemodel's (cout, cin, k, k) floats; `bias`, `bn_scale`, `bn_shift`: cout
// floats or NULL, no BN without a scale) into the one layout its path reads and uploads them.  The caller has set the
// shape fields and chosen the path (op.split, op.use_tc); a tensor-core op also gets its plan from `in` to `out` (split:
// the float input, whose half planes a_split it allocates).  `act`: the activation type (fp16 rounds the SIMT weights
// through half).
void prepare_conv(Op& op, DType act, const float* w, const float* bias, const float* bn_scale, const float* bn_shift,
                  const TensorView& in, const TensorView& out);
// one run of convolution `op` from `in` to `out` on `s`: the split-operand mode's hi / lo pass and the plan, or the SIMT kernel
void launch_conv(const Op& op, const TensorView& in, const TensorView& out, cudaStream_t s);
// the [hi Cin | lo Cin] half planes of float tensor `v` that a split-operand convolution reads (p unset)
TensorView split_view(TensorView v);

// conv_tc.cu -- wgmma implicit-GEMM convolution
bool conv_tc_supported(const Op& op, const TensorView& in, const TensorView& out);
std::shared_ptr<ConvTcPlan> conv_tc_plan(const Op& op, const TensorView& in, const TensorView& out, const void* w_tc);
void conv_tc_launch(const ConvTcPlan& plan, cudaStream_t s);
// input rows whose MMAs the plan's kernel runs per output row: > 1 for the tap-row-stacked float-logits kernel (warm-up rows)
double conv_tc_rows_ratio(const ConvTcPlan& plan);
// fuses the sampling Dropout that follows the convolution in place into its epilogue
// (sample0: global MC sample index of the batch's image 0, so that a shard handle draws the masks of its own samples)
void conv_tc_set_dropout(ConvTcPlan& plan, uint64_t seed, const uint64_t* frame_dev, int layer, float scale, int sample0);
// fuses the max-unpool (Upsample) that consumes the convolution's output into its epilogue; `out_2h_2w` is the
// unpooled tensor the convolution then writes instead of its own output.  k_conv_tn plans have no such epilogue: their
// output is unpooled by its consumer (conv_tc_set_unpool_input) or by the unpool kernel.
bool conv_tc_can_fuse_unpool(const ConvTcPlan& plan);
void conv_tc_set_unpool(ConvTcPlan& plan, const uint8_t* mask, int mask_n, void* out_2h_2w);
// makes a 7x7 float-logits (k_conv_stack) or 64-wide half (k_conv_tn) plan read the max-unpool of `pooled` ([n][h][w][64]
// half, the plan's input being 2h x 2w) by `mask` (same layout, batch mask_n) instead of its input tensor: the unpool is
// done as the halo rows are loaded
bool conv_tc_can_unpool_input(const ConvTcPlan& plan);
void conv_tc_set_unpool_input(ConvTcPlan& plan, const void* pooled, const uint8_t* mask, int mask_n, int h, int w);
// fuses the 2x2/2 max pool (+ argmax mask) that consumes the convolution's output into its epilogue
bool conv_tc_can_fuse_pool(const ConvTcPlan& plan);
void conv_tc_set_pool(ConvTcPlan& plan, void* pooled, uint8_t* mask);
// host-side weight layout of the split-operand fp32 mode: [tap][cout_p][3 cin_p] half + the accumulator scale 2^-s
std::vector<__half> conv_tc_split_weights(const float* w_cout_cin_k_k, int cout, int cin, int K, int cout_p, int cin_p, float* acc_scale);
// The composed classifier: conv (64 -> 64, 7x7, no BN / ReLU) followed by the 1x1 classifier run as ONE 64 -> 16 convolution
// with composed weights; logits come straight from the accumulators.  wc = [n_cls][64], bc = [n_cls] or NULL (host).
bool conv_tc_can_compose_classifier(const ConvTcPlan& plan);
void conv_tc_set_composed_classifier(ConvTcPlan& plan, const Op& conv, const float* wc, const float* bc, int n_cls, float* logits);

}  // namespace sivo
