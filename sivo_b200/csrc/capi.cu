// extern "C" boundary of libsivo_b200.so (include/sivo_b200.h).  No C++ type, exception or abort crosses it.
#include <cuda_fp16.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <string>

#include "frame_ops.h"
#include "segnet.h"
#include "vocabulary.h"

namespace sivo {
namespace {
thread_local std::string g_last_error;
}
void set_last_error(const std::string& m) { g_last_error = m; }
}  // namespace sivo

using namespace sivo;

struct sivo_segnet { SegNet* impl; };
struct sivo_orb { Orb* impl; };
struct sivo_vocabulary { Vocabulary* impl; };
struct sivo_pnp { Pnp* impl; };

extern "C" {

const char* sivo_last_error(void) { return g_last_error.c_str(); }
const char* sivo_version(void) { return "sivo_b200 0.1 (sm_90a)"; }

int sivo_segnet_create_ex(const char* prototxt, const char* caffemodel, const sivo_segnet_options* opt, sivo_segnet_t** out) {
  return guarded([&] {
    if (!out) fail(SIVO_EINVAL, "null output handle");
    *out = nullptr;
    sivo_segnet_options o{};
    if (opt) o = *opt;
    auto* impl = new SegNet(prototxt ? prototxt : "", caffemodel ? caffemodel : "", o);
    *out = new sivo_segnet{impl};
  });
}

int sivo_segnet_create_shard(const char* prototxt, const char* caffemodel, const sivo_segnet_options* opt, int sample_begin,
                             int sample_count, sivo_segnet_t** out) {
  return guarded([&] {
    if (!out) fail(SIVO_EINVAL, "null output handle");
    *out = nullptr;
    if (sample_begin < 0 || sample_count < 1)
      fail(SIVO_EINVAL, "sample range: begin %d must be >= 0 and count %d >= 1", sample_begin, sample_count);
    sivo_segnet_options o{};
    if (opt) o = *opt;
    auto* impl = new SegNet(prototxt ? prototxt : "", caffemodel ? caffemodel : "", o, sample_begin, sample_count);
    *out = new sivo_segnet{impl};
  });
}

int sivo_segnet_samples(const sivo_segnet_t* h, int* sample_begin, int* sample_count, int* T_total) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    if (sample_begin) *sample_begin = h->impl->sample_begin();
    if (sample_count) *sample_count = h->impl->sample_count();
    if (T_total) *T_total = h->impl->T();
  });
}

int sivo_segnet_run_partial_device(sivo_segnet_t* h, const uint8_t* bgr_device, double* sum_device, void* stream) {
  return guarded([&] {
    if (!h || !bgr_device || !sum_device) fail(SIVO_EINVAL, "null handle, image or sum buffer");
    h->impl->run_partial(bgr_device, sum_device, static_cast<cudaStream_t>(stream));
  });
}

int sivo_segnet_finalize_device(sivo_segnet_t* h, const double* sum_device, uint8_t* classes_device, double* confidence_device,
                                double* entropy_device, float* confidence_f32_device, float* entropy_f32_device, void* stream) {
  return guarded([&] {
    if (!h || !sum_device) fail(SIVO_EINVAL, "null handle or sum buffer");
    h->impl->finalize(sum_device, classes_device, confidence_device, entropy_device, confidence_f32_device, entropy_f32_device,
                      static_cast<cudaStream_t>(stream));
  });
}

int sivo_segnet_variance(sivo_segnet_t* h, const uint8_t* classes, double* variance) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    h->impl->variance_host(classes, variance);
  });
}

int sivo_segnet_variance_device(sivo_segnet_t* h, const uint8_t* classes_device, double* variance_device, void* stream) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    h->impl->variance_device(classes_device, variance_device, static_cast<cudaStream_t>(stream));
  });
}

int sivo_segnet_variance_partial_device(sivo_segnet_t* h, const uint8_t* classes_device, double* moments_device, void* stream) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    h->impl->variance_partial(classes_device, moments_device, static_cast<cudaStream_t>(stream));
  });
}

int sivo_segnet_variance_finalize_device(sivo_segnet_t* h, const double* moments_device, double* variance_device, void* stream) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    h->impl->variance_finalize(moments_device, variance_device, static_cast<cudaStream_t>(stream));
  });
}

int sivo_segnet_create(const char* prototxt, const char* caffemodel, int device, uint64_t seed, sivo_segnet_t** out) {
  sivo_segnet_options o{};
  o.device = device;
  o.seed = seed;
  // knobs with no slot in the reference's constructor come from the environment (the C++ shim calls this entry point):
  // SIVO_B200_PRECISION = fp16 (default: the fast mode) | fp32 (strict: split-operand tensor-core convolutions, fp32 activations);
  // SIVO_B200_ENGINE = auto | simt | tcgen05
  if (const char* e = std::getenv("SIVO_B200_PRECISION")) o.precision = (std::string(e) == "fp32") ? SIVO_PRECISION_FP32 : SIVO_PRECISION_FP16;
  if (const char* e = std::getenv("SIVO_B200_ENGINE"))
    o.engine = std::string(e) == "simt" ? SIVO_ENGINE_SIMT : std::string(e) == "tcgen05" ? SIVO_ENGINE_TCGEN05 : SIVO_ENGINE_AUTO;
  return sivo_segnet_create_ex(prototxt, caffemodel, &o, out);
}

int sivo_segnet_geometry(const sivo_segnet_t* h, int* width, int* height, int* T, int* n_classes) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    if (width) *width = h->impl->width();
    if (height) *height = h->impl->height();
    if (T) *T = h->impl->T();
    if (n_classes) *n_classes = h->impl->classes();
  });
}

int sivo_segnet_set_frame(sivo_segnet_t* h, uint64_t frame) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    h->impl->set_frame(frame);
  });
}

int sivo_segnet_set_profiling(sivo_segnet_t* h, int on) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    h->impl->set_profiling(on != 0);
  });
}

int sivo_segnet_run(sivo_segnet_t* h, const uint8_t* bgr, int rows, int cols, size_t stride, uint8_t* classes,
                    double* confidence, double* entropy) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    h->impl->run_host(bgr, rows, cols, stride, classes, confidence, entropy);
  });
}

int sivo_segnet_run_device(sivo_segnet_t* h, const uint8_t* bgr_device, uint8_t* classes_device, double* confidence_device,
                           double* entropy_device, void* stream) {
  return guarded([&] {
    if (!h || !bgr_device) fail(SIVO_EINVAL, "null handle or image");
    h->impl->run_device(bgr_device, classes_device, confidence_device, entropy_device, static_cast<cudaStream_t>(stream));
  });
}

int sivo_segnet_set_record_outputs(sivo_segnet_t* h, uint8_t* classes_device, float* confidence_f32_device, float* entropy_f32_device) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    h->impl->set_record_outputs(classes_device, confidence_f32_device, entropy_f32_device);
  });
}

int sivo_segnet_run_device_maps(sivo_segnet_t* h, const uint8_t* bgr_device, uint8_t* classes_device, double* confidence_device,
                                double* entropy_device, float* confidence_f32_device, float* entropy_f32_device, void* stream) {
  return guarded([&] {
    if (!h || !bgr_device) fail(SIVO_EINVAL, "null handle or image");
    h->impl->run_device(bgr_device, classes_device, confidence_device, entropy_device, static_cast<cudaStream_t>(stream),
                        confidence_f32_device, entropy_f32_device);
  });
}

int sivo_segnet_blob(sivo_segnet_t* h, const char* name, float* out, size_t cap, int* n, int* c, int* hh, int* ww) {
  return guarded([&] {
    if (!h || !name) fail(SIVO_EINVAL, "null handle or name");
    h->impl->blob(name, out, cap, n, c, hh, ww);
  });
}

int sivo_segnet_last_timing(const sivo_segnet_t* h, float* conv_ms, float* other_ms, float* reduce_ms, float* total_ms,
                            int* launches) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    if (conv_ms) *conv_ms = h->impl->conv_ms;
    if (other_ms) *other_ms = h->impl->other_ms;
    if (reduce_ms) *reduce_ms = h->impl->reduce_ms;
    if (total_ms) *total_ms = h->impl->total_ms;
    if (launches) *launches = h->impl->launches;
  });
}

int sivo_segnet_semantic_keys(sivo_segnet_t* h, const sivo_keypoint* kps, int n, int max_static_class, uint8_t* kp_class, double* kp_conf,
                              double* kp_entropy, int* keep_idx, int* n_keep) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    h->impl->semantic_keys(kps, n, max_static_class, kp_class, kp_conf, kp_entropy, keep_idx, n_keep);
  });
}

int sivo_segnet_semantic_keys_device(sivo_segnet_t* h, const sivo_keypoint* kps_device, const long long* count_device, int cap,
                                     int max_static_class, uint8_t* kp_class_device, double* kp_conf_device, double* kp_entropy_device,
                                     int* keep_idx_device, long long* n_keep_device, void* stream) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    h->impl->semantic_keys_device(kps_device, count_device, cap, max_static_class, kp_class_device, kp_conf_device, kp_entropy_device,
                                  keep_idx_device, n_keep_device, static_cast<cudaStream_t>(stream));
  });
}

int sivo_segnet_op_timing(const sivo_segnet_t* h, int index, char* name, size_t cap, float* ms, double* flops, int* n_ops) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    const int n = static_cast<int>(h->impl->n_ops());
    if (n_ops) *n_ops = n;
    if (index < 0) return;  // count query
    if (index >= n) fail(SIVO_ERANGE, "op index %d out of range (%d launches)", index, n);
    const Op& op = h->impl->op_at(index);
    if (name && cap) snprintf(name, cap, "%s", op.layer.c_str());
    if (ms) *ms = static_cast<size_t>(index) < h->impl->op_ms.size() ? h->impl->op_ms[index] : 0.f;
    if (flops) *flops = op.kind == Op::Conv ? op.flops : 0.0;
  });
}

int sivo_segnet_op_flops_executed(const sivo_segnet_t* h, int index, double* flops) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    const int n = static_cast<int>(h->impl->n_ops());
    if (index < 0 || index >= n) fail(SIVO_ERANGE, "op index %d out of range (%d launches)", index, n);
    const Op& op = h->impl->op_at(index);
    if (flops) *flops = op.kind == Op::Conv ? op.flops_exec : 0.0;
  });
}

int sivo_segnet_flops(const sivo_segnet_t* h, double* dedup, double* naive) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    if (dedup) *dedup = h->impl->flops_dedup;
    if (naive) *naive = h->impl->flops_naive;
  });
}

void sivo_segnet_destroy(sivo_segnet_t* h) {
  if (!h) return;
  delete h->impl;
  delete h;
}

// ---------------------------------------------------------------------------------------- ORB
int sivo_orb_create(int nfeatures, float scale_factor, int nlevels, int ini_th_fast, int min_th_fast, int device,
                    sivo_orb_t** out) {
  return guarded([&] {
    if (!out) fail(SIVO_EINVAL, "null output handle");
    *out = nullptr;
    auto* impl = new Orb(nfeatures, scale_factor, nlevels, ini_th_fast, min_th_fast, device);
    *out = new sivo_orb{impl};
  });
}

int sivo_orb_tables(const sivo_orb_t* h, float* scale, float* inv_scale, float* sigma2, float* inv_sigma2, int* per_level) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    const OrbTables& t = h->impl->tables();
    size_t n = t.scale.size();
    if (scale) memcpy(scale, t.scale.data(), n * sizeof(float));
    if (inv_scale) memcpy(inv_scale, t.inv_scale.data(), n * sizeof(float));
    if (sigma2) memcpy(sigma2, t.sigma2.data(), n * sizeof(float));
    if (inv_sigma2) memcpy(inv_sigma2, t.inv_sigma2.data(), n * sizeof(float));
    if (per_level) memcpy(per_level, t.per_level.data(), n * sizeof(int));
  });
}

int sivo_orb_run(sivo_orb_t* h, const uint8_t* gray, int rows, int cols, size_t stride, sivo_keypoint* kps, int cap, int* n,
                 uint8_t* desc32, uint8_t* const* pyramid_levels, const size_t* pyramid_strides) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    h->impl->run(gray, rows, cols, stride, kps, cap, n, desc32, pyramid_levels, pyramid_strides);
  });
}

int sivo_orb_run_device_input(sivo_orb_t* h, const uint8_t* gray_device, int rows, int cols, size_t pitch, sivo_keypoint* kps,
                              int cap, int* n, uint8_t* desc32) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    h->impl->run(gray_device, rows, cols, pitch, kps, cap, n, desc32, nullptr, nullptr, true);
  });
}

int sivo_orb_enqueue_device(sivo_orb_t* h, const uint8_t* gray_device, int rows, int cols, size_t pitch, sivo_keypoint* kps_device,
                            uint8_t* desc32_device, long long* count_device) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    h->impl->enqueue_device(gray_device, rows, cols, pitch, kps_device, desc32_device, count_device);
  });
}

int sivo_orb_stream_wait(sivo_orb_t* h, void* consumer_cuda_stream) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    h->impl->stream_wait(static_cast<cudaStream_t>(consumer_cuda_stream));
  });
}

int sivo_orb_wait_for_stream(sivo_orb_t* h, void* producer_cuda_stream) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    h->impl->wait_for_stream(static_cast<cudaStream_t>(producer_cuda_stream));
  });
}

int sivo_orb_wait_event(sivo_orb_t* h, void* cuda_event) {
  return guarded([&] {
    if (!h || !cuda_event) fail(SIVO_EINVAL, "null argument");
    h->impl->wait_event(static_cast<cudaEvent_t>(cuda_event));
  });
}

int sivo_orb_device_status(sivo_orb_t* h, int* level_mask) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    const int m = h->impl->device_tree_status();
    if (level_mask) *level_mask = m;
  });
}

int sivo_orb_has_device_tree(const sivo_orb_t* h, int* yes) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    if (yes) *yes = h->impl->device_tree() ? 1 : 0;
  });
}

int sivo_orb_capacity(const sivo_orb_t* h, int* max_keypoints) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    if (max_keypoints) *max_keypoints = h->impl->capacity();
  });
}

int sivo_orb_level_size(const sivo_orb_t* h, int rows, int cols, int level, int* level_w, int* level_h) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    h->impl->level_size(rows, cols, level, level_w, level_h);
  });
}

int sivo_orb_candidates(const sivo_orb_t* h, int level, int* xs, int* ys, int* resp, int cap, int* n) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    h->impl->candidates(level, xs, ys, resp, cap, n);
  });
}

int sivo_orb_last_timing(const sivo_orb_t* h, float* device_ms, float* host_tree_ms, int* launches) {
  return guarded([&] {
    if (!h) fail(SIVO_EINVAL, "null handle");
    if (device_ms) *device_ms = h->impl->device_ms;
    if (host_tree_ms) *host_tree_ms = h->impl->tree_ms;
    if (launches) *launches = h->impl->launches;
  });
}

void sivo_orb_destroy(sivo_orb_t* h) {
  if (!h) return;
  delete h->impl;
  delete h;
}

int sivo_orb_distribute(const float* xs, const float* ys, const float* resp, int n, int min_x, int max_x, int min_y, int max_y,
                        int n_target, int* keep, int cap) {
  int count = 0;
  int rc = guarded([&] {
    if (n > 0 && (!xs || !ys || !resp)) fail(SIVO_EINVAL, "null keypoint arrays");
    if (max_x <= min_x || max_y <= min_y) fail(SIVO_EINVAL, "empty distribution rectangle");
    std::vector<int> k = orb_distribute(xs, ys, resp, n, min_x, max_x, min_y, max_y, n_target);
    if (static_cast<int>(k.size()) > cap) fail(SIVO_ERANGE, "%zu kept keypoints, buffer holds %d", k.size(), cap);
    if (keep) memcpy(keep, k.data(), k.size() * sizeof(int));
    count = static_cast<int>(k.size());
  });
  return rc == SIVO_OK ? count : rc;
}

int sivo_dbg_orb_distribute_device(int device, const int* xs, const int* ys, const int* resp, int n, int min_x, int max_x, int min_y,
                                   int max_y, int n_target, int* out_x, int* out_y, int* out_resp, int cap) {
  int count = 0;
  int rc = guarded([&] {
    if (n > 0 && (!xs || !ys || !resp)) fail(SIVO_EINVAL, "null keypoint arrays");
    if (max_x <= min_x || max_y <= min_y) fail(SIVO_EINVAL, "empty distribution rectangle");
    SIVO_CUDA(cudaSetDevice(device));
    orb_tree_configure();
    OrbTreeParams prm{};
    int n_ini = static_cast<int>(std::round(static_cast<float>(max_x - min_x) / (max_y - min_y)));
    if (n_ini < 1) n_ini = 1;
    prm.n_target[0] = n_target; prm.n_ini[0] = n_ini; prm.height[0] = max_y - min_y;
    prm.hx[0] = static_cast<float>(max_x - min_x) / n_ini;
    prm.scale[0] = 1.f; prm.size[0] = 31.f; prm.min_b = 0;
    std::vector<uint32_t> packed(std::max(n, 1));
    for (int i = 0; i < n; ++i) {
      if (xs[i] < 0 || xs[i] > 4095 || ys[i] < 0 || ys[i] > 4095 || resp[i] < 0 || resp[i] > 255) fail(SIVO_EINVAL, "key %d out of range", i);
      packed[i] = static_cast<uint32_t>(xs[i]) | (static_cast<uint32_t>(ys[i]) << 12) | (static_cast<uint32_t>(resp[i]) << 24);
    }
    const int off[2] = {0, n};
    DevBuf d_cand(packed.size() * 4), d_off(sizeof off), d_sel(static_cast<size_t>(kTreeSelCap) * 4), d_cnt(2 * sizeof(int));
    SIVO_CUDA(cudaMemcpy(d_cand.p, packed.data(), packed.size() * 4, cudaMemcpyHostToDevice));
    SIVO_CUDA(cudaMemcpy(d_off.p, off, sizeof off, cudaMemcpyHostToDevice));
    SIVO_CUDA(cudaMemset(d_cnt.p, 0, 2 * sizeof(int)));
    orb_launch_distribute(d_cand.as<uint32_t>(), d_off.as<int>(), nullptr, nullptr, prm, 1, d_sel.as<uint32_t>(), d_cnt.as<int>(), d_cnt.as<int>() + 1, nullptr);
    int ce[2] = {0, 0};
    SIVO_CUDA(cudaMemcpy(ce, d_cnt.p, sizeof ce, cudaMemcpyDeviceToHost));
    if (ce[1]) fail(SIVO_ERANGE, "input exceeds the device quad tree's capacity");
    if (ce[0] > cap) fail(SIVO_ERANGE, "%d kept keypoints, buffer holds %d", ce[0], cap);
    std::vector<uint32_t> sel(std::max(ce[0], 1));
    SIVO_CUDA(cudaMemcpy(sel.data(), d_sel.p, static_cast<size_t>(ce[0]) * 4, cudaMemcpyDeviceToHost));
    for (int i = 0; i < ce[0]; ++i) {
      if (out_x) out_x[i] = static_cast<int>(sel[i] & 0xFFF);
      if (out_y) out_y[i] = static_cast<int>((sel[i] >> 12) & 0xFFF);
      if (out_resp) out_resp[i] = static_cast<int>(sel[i] >> 24);
    }
    count = ce[0];
  });
  return rc == SIVO_OK ? count : rc;
}

int sivo_stereo_hamming(int device, const sivo_keypoint* left, const uint8_t* desc_left, int n_left, const sivo_keypoint* right,
                        const uint8_t* desc_right, int n_right, const float* scale_factors, int nlevels, int rows, float min_d,
                        float max_d, int* best_idx, int* best_dist) {
  return guarded([&] {
    if (!scale_factors || !best_idx || !best_dist || (n_left && (!left || !desc_left)) || (n_right && (!right || !desc_right)))
      fail(SIVO_EINVAL, "null argument");
    stereo_hamming(device, left, desc_left, n_left, right, desc_right, n_right, scale_factors, nlevels, rows, min_d, max_d,
                   best_idx, best_dist);
  });
}

int sivo_hamming_best2(int device, const uint8_t* query_desc, int n_query, const uint8_t* train_desc, int n_train,
                       const int* cand_offsets, const int* cand_idx, const int* train_level, int* out5) {
  return guarded([&] {
    if (!out5 || !cand_offsets || (n_query && !query_desc) || (n_train && !train_desc) || (n_query > 0 && cand_offsets[n_query] && !cand_idx))
      fail(SIVO_EINVAL, "null argument");
    hamming_best2(device, query_desc, n_query, train_desc, n_train, cand_offsets, cand_idx, train_level, out5);
  });
}

int sivo_stereo_match(const sivo_orb_t* left, const sivo_orb_t* right, const sivo_keypoint* kp_left, const uint8_t* desc_left,
                      int n_left, const sivo_keypoint* kp_right, const uint8_t* desc_right, int n_right, float mb, float mbf,
                      float* u_right, float* depth) {
  return guarded([&] {
    if (!left || !right || !u_right || !depth || (n_left && (!kp_left || !desc_left)) || (n_right && (!kp_right || !desc_right)))
      fail(SIVO_EINVAL, "null argument");
    stereo_match(*left->impl, *right->impl, kp_left, desc_left, n_left, kp_right, desc_right, n_right, mb, mbf, u_right, depth);
  });
}

int sivo_stereo_match_device(sivo_orb_t* left, sivo_orb_t* right, const sivo_keypoint* kp_left_device, const uint8_t* desc_left_device,
                             const int* keep_idx_device, const long long* n_left_device, const sivo_keypoint* kp_right_device,
                             const uint8_t* desc_right_device, const long long* n_right_device, float mb, float mbf, float* u_right_device,
                             float* depth_device, void* stream) {
  return guarded([&] {
    if (!left || !right || !kp_left_device || !desc_left_device || !n_left_device || !kp_right_device || !desc_right_device ||
        !n_right_device || !u_right_device || !depth_device)
      fail(SIVO_EINVAL, "null argument");
    stereo_match_device(*left->impl, *right->impl, kp_left_device, desc_left_device, keep_idx_device, n_left_device, kp_right_device,
                        desc_right_device, n_right_device, mb, mbf, u_right_device, depth_device, static_cast<cudaStream_t>(stream));
  });
}

int sivo_dbg_stereo_median_cut(int device, const int* sad, int n, float* u, float* z) {
  return guarded([&] {
    if (n > 0 && (!sad || !u || !z)) fail(SIVO_EINVAL, "null argument");
    stereo_median_cut(device, sad, n, u, z);
  });
}

// ---------------------------------------------------------------------------------------- information selection
int sivo_info_select(const sivo_orb_t* left, const sivo_keypoint* kps, const float* depth, const double* entropy, int n,
                     const sivo_info_camera* cam, double threshold, float* world, double* reduction, int* selected, int* n_selected) {
  return guarded([&] {
    if (!left || !cam || n < 0 || (n && (!kps || !depth || !entropy))) fail(SIVO_EINVAL, "info_select: null argument or n < 0");
    info_select(*left->impl, kps, depth, entropy, n, *cam, threshold, world, reduction, selected, n_selected);
  });
}

int sivo_info_select_device(const sivo_orb_t* left, const sivo_keypoint* kps_device, const double* kp_entropy_device,
                            const int* keep_idx_device, const long long* n_keep_device, const float* depth_device,
                            const sivo_info_camera* cam, double threshold, float* world_device, double* reduction_device,
                            int* selected_device, long long* n_selected_device, void* stream) {
  return guarded([&] {
    if (!left || !kps_device || !kp_entropy_device || !n_keep_device || !depth_device || !cam) fail(SIVO_EINVAL, "info_select: null argument");
    info_select_device(*left->impl, kps_device, kp_entropy_device, keep_idx_device, n_keep_device, depth_device, *cam, threshold, world_device,
                       reduction_device, selected_device, n_selected_device, static_cast<cudaStream_t>(stream));
  });
}

int sivo_dbg_info_terms(const sivo_orb_t* left, const sivo_keypoint* kps, const float* depth, int n, const sivo_info_camera* cam,
                        float* world, double* det_state, double* det_meas, double* det_joint) {
  return guarded([&] {
    if (!left || !cam || n < 0 || (n && (!kps || !depth))) fail(SIVO_EINVAL, "info_terms: null argument or n < 0");
    info_terms(*left->impl, kps, depth, n, *cam, world, det_state, det_meas, det_joint);
  });
}

// ---------------------------------------------------------------------------------------- projection searches
int sivo_search_local_points_device(const sivo_orb_t* left, const sivo_keypoint* kps_device, const uint8_t* desc_device,
                                    const int* keep_idx_device, const long long* n_keep_device, const float* u_right_device,
                                    const uint8_t* blocked_device, const sivo_map_point* points_device, int n_points,
                                    const sivo_track_frame* frame, float th, float nnratio, uint8_t* in_view_device, int* match_device,
                                    long long* n_matches_device, void* stream) {
  return guarded([&] {
    if (!left || !kps_device || !desc_device || !n_keep_device || !u_right_device || !frame || (n_points > 0 && !points_device))
      fail(SIVO_EINVAL, "search_local_points: null argument");
    search_local_points_device(*left->impl, kps_device, desc_device, keep_idx_device, n_keep_device, u_right_device, blocked_device,
                               points_device, n_points, *frame, th, nnratio, in_view_device, match_device, n_matches_device,
                               static_cast<cudaStream_t>(stream));
  });
}

int sivo_search_last_frame_device(const sivo_orb_t* left, const sivo_keypoint* kps_device, const uint8_t* desc_device,
                                  const int* keep_idx_device, const long long* n_keep_device, const float* u_right_device,
                                  const sivo_map_point* points_device, int n_points, const sivo_track_frame* frame, const float* Rlw,
                                  const float* tlw, float th, int* match_device, long long* n_matches_device, void* stream) {
  return guarded([&] {
    if (!left || !kps_device || !desc_device || !n_keep_device || !u_right_device || !frame || !Rlw || !tlw ||
        (n_points > 0 && !points_device))
      fail(SIVO_EINVAL, "search_last_frame: null argument");
    search_last_frame_device(*left->impl, kps_device, desc_device, keep_idx_device, n_keep_device, u_right_device, points_device, n_points,
                             *frame, Rlw, tlw, th, match_device, n_matches_device, static_cast<cudaStream_t>(stream));
  });
}

int sivo_search_local_points(const sivo_orb_t* left, const sivo_keypoint* kps, const uint8_t* desc, const float* u_right,
                             const uint8_t* blocked, int n, const sivo_map_point* points, int n_points, const sivo_track_frame* frame,
                             float th, float nnratio, uint8_t* in_view, int* match, int* n_matches) {
  return guarded([&] {
    if (!left || !frame || n < 0 || (n && (!kps || !desc || !u_right)) || (n_points > 0 && !points))
      fail(SIVO_EINVAL, "search_local_points: null argument or n < 0");
    search_local_points(*left->impl, kps, desc, u_right, blocked, n, points, n_points, *frame, th, nnratio, in_view, match, n_matches);
  });
}

int sivo_search_last_frame(const sivo_orb_t* left, const sivo_keypoint* kps, const uint8_t* desc, const float* u_right, int n,
                           const sivo_map_point* points, int n_points, const sivo_track_frame* frame, const float* Rlw,
                           const float* tlw, float th, int* match, int* n_matches) {
  return guarded([&] {
    if (!left || !frame || !Rlw || !tlw || n < 0 || (n && (!kps || !desc || !u_right)) || (n_points > 0 && !points))
      fail(SIVO_EINVAL, "search_last_frame: null argument or n < 0");
    search_last_frame(*left->impl, kps, desc, u_right, n, points, n_points, *frame, Rlw, tlw, th, match, n_matches);
  });
}

int sivo_dbg_features_in_area(const sivo_orb_t* left, const sivo_keypoint* kps, int n, float min_x, float max_x, float min_y,
                              float max_y, const float* xyr, const int* levels, int n_query, int* offsets, int* idx, int idx_cap) {
  return guarded([&] {
    if (!left || !offsets || n < 0 || n_query < 0 || (n && !kps) || (n_query && (!xyr || !levels)) || (idx_cap > 0 && !idx))
      fail(SIVO_EINVAL, "features_in_area: null argument or negative count");
    sivo_track_frame f{};
    f.min_x = min_x; f.max_x = max_x; f.min_y = min_y; f.max_y = max_y;
    features_in_area(*left->impl, kps, n, f, xyr, levels, n_query, offsets, idx, idx_cap);
  });
}

// ---------------------------------------------------------------------------------------- frame pose
int sivo_pose_optimize_device(const sivo_orb_t* left, const sivo_keypoint* kps_device, const int* keep_idx_device,
                              const long long* n_keep_device, const float* u_right_device, const float* xw_device, float fx, float fy,
                              float cx, float cy, float mbf, const float* Tcw_in_device, sivo_pose_result* result_device,
                              uint8_t* outlier_device, void* stream) {
  return guarded([&] {
    if (!left || !kps_device || !n_keep_device || !u_right_device || !xw_device || !Tcw_in_device || !result_device)
      fail(SIVO_EINVAL, "pose_optimize: null argument");
    pose_optimize_device(*left->impl, kps_device, keep_idx_device, n_keep_device, u_right_device, xw_device, fx, fy, cx, cy, mbf,
                         Tcw_in_device, result_device, outlier_device, static_cast<cudaStream_t>(stream));
  });
}

int sivo_pose_gather_device(const sivo_orb_t* left, const int* match_device, const long long* n_keep_device,
                            const sivo_map_point* points_device, int n_points, float* xw_device, void* stream) {
  return guarded([&] {
    if (!left || !match_device || !n_keep_device || !xw_device || (n_points > 0 && !points_device))
      fail(SIVO_EINVAL, "pose_gather: null argument");
    pose_gather_device(*left->impl, match_device, n_keep_device, points_device, n_points, xw_device, static_cast<cudaStream_t>(stream));
  });
}

int sivo_pose_optimize(const sivo_orb_t* left, const sivo_keypoint* kps, const float* u_right, const float* xw, int n, float fx,
                       float fy, float cx, float cy, float mbf, const float* Tcw_in, sivo_pose_result* result, uint8_t* outlier) {
  return guarded([&] {
    if (!left || !Tcw_in || !result || n < 0 || (n && (!kps || !u_right || !xw))) fail(SIVO_EINVAL, "pose_optimize: null argument or n < 0");
    pose_optimize(*left->impl, kps, u_right, xw, n, fx, fy, cx, cy, mbf, Tcw_in, result, outlier);
  });
}

int sivo_dbg_pose_system(const sivo_orb_t* left, const sivo_keypoint* kps, const float* u_right, const float* xw, int n, float fx,
                         float fy, float cx, float cy, float mbf, const double* pose7, int robust_stereo, const uint8_t* level1,
                         double* err, double* chi2, double* rho, double* jac, double* H, double* b, double* chi) {
  return guarded([&] {
    if (!left || !pose7 || n < 0 || (n && (!kps || !u_right || !xw))) fail(SIVO_EINVAL, "pose_system: null argument or n < 0");
    pose_system(*left->impl, kps, u_right, xw, n, fx, fy, cx, cy, mbf, pose7, robust_stereo, level1, err, chi2, rho, jac, H, b, chi);
  });
}

int sivo_dbg_pose_trace(const sivo_orb_t* left, const sivo_keypoint* kps, const float* u_right, const float* xw, int n, float fx,
                        float fy, float cx, float cy, float mbf, const float* Tcw_in, sivo_pose_result* result, uint8_t* outlier,
                        sivo_pose_trace_rec* trace, int trace_cap) {
  int n_rec = 0;
  const int rc = guarded([&] {
    if (!left || !Tcw_in || !result || n < 0 || (n && (!kps || !u_right || !xw))) fail(SIVO_EINVAL, "pose_trace: null argument or n < 0");
    n_rec = pose_trace(*left->impl, kps, u_right, xw, n, fx, fy, cx, cy, mbf, Tcw_in, result, outlier, trace, trace_cap);
  });
  return rc ? rc : n_rec;
}

int sivo_dbg_pose_se3(int device, int n, const float* T, const double* d, double* se3, double* up, double* tv, sivo_pose_result* res) {
  return guarded([&] { pose_se3(device, n, T, d, se3, up, tv, res); });
}

// ---------------------------------------------------------------------------------------- keyframe map points
int sivo_keyframe_gather_device(const sivo_orb_t* left, const sivo_keypoint* kps_device, const uint8_t* desc_device,
                                const int* keep_idx_device, const long long* n_keep_device, const float* u_right_device,
                                const float* depth_device, const uint8_t* kp_class_device, const double* kp_conf_device,
                                const double* kp_entropy_device, sivo_keypoint* out_kps, uint8_t* out_desc, float* out_u_right,
                                float* out_depth, uint8_t* out_class, double* out_conf, double* out_entropy, long long* out_count,
                                void* stream) {
  return guarded([&] {
    if (!left || !kps_device || !desc_device || !n_keep_device || !u_right_device || !depth_device || !kp_class_device || !kp_conf_device ||
        !kp_entropy_device || !out_kps || !out_desc || !out_u_right || !out_depth || !out_class || !out_conf || !out_entropy || !out_count)
      fail(SIVO_EINVAL, "keyframe_gather: null argument");
    keyframe_gather_device(*left->impl, kps_device, desc_device, keep_idx_device, n_keep_device, u_right_device, depth_device, kp_class_device,
                           kp_conf_device, kp_entropy_device, out_kps, out_desc, out_u_right, out_depth, out_class, out_conf, out_entropy,
                           out_count, static_cast<cudaStream_t>(stream));
  });
}

int sivo_create_map_points_device(const sivo_orb_t* left, const sivo_keyframe_keys* kf1, const sivo_keyframe_keys* neighbours,
                                  int n_neighbours, const sivo_mapping_params* params, int* created_nb_device,
                                  int* created_idx_device, float* world_device, int* created_list_device, long long* n_created_device,
                                  void* stream) {
  return guarded([&] {
    if (!left || !kf1 || !params) fail(SIVO_EINVAL, "create_map_points: null argument");
    create_map_points_device(*left->impl, *kf1, neighbours, n_neighbours, *params, created_nb_device, created_idx_device, world_device,
                             created_list_device, n_created_device, static_cast<cudaStream_t>(stream));
  });
}

int sivo_create_map_points(const sivo_orb_t* left, const sivo_keyframe_keys* kf1, const sivo_keyframe_keys* neighbours, int n_neighbours,
                           const sivo_mapping_params* params, int* created_nb, int* created_idx, float* world, int* created_list,
                           long long* n_created) {
  return guarded([&] {
    if (!left || !kf1 || !params) fail(SIVO_EINVAL, "create_map_points: null argument");
    create_map_points_host(*left->impl, *kf1, neighbours, n_neighbours, *params, nullptr, nullptr, nullptr, created_nb, created_idx, world,
                           created_list, n_created);
  });
}

int sivo_dbg_create_map_points(const sivo_orb_t* left, const sivo_keyframe_keys* kf1, const sivo_keyframe_keys* neighbours,
                               int n_neighbours, const sivo_mapping_params* params, int* match, int* stage, double* reduction,
                               int* created_nb, int* created_idx, float* world, int* created_list, long long* n_created) {
  return guarded([&] {
    if (!left || !kf1 || !params || !match || !stage || !reduction) fail(SIVO_EINVAL, "create_map_points: null argument");
    create_map_points_host(*left->impl, *kf1, neighbours, n_neighbours, *params, match, stage, reduction, created_nb, created_idx, world,
                           created_list, n_created);
  });
}

// ---------------------------------------------------------------------------------------- keyframe Fuse
int sivo_fuse_device(const sivo_orb_t* left, const sivo_keyframe_keys* targets, int n_targets, const sivo_fuse_camera* cam,
                     const sivo_map_point* points_device, int n_points, float th, int* match_device, int* dist_device, void* stream) {
  return guarded([&] {
    if (!left || !cam || (n_points > 0 && !points_device) || (n_targets > 0 && n_points > 0 && !match_device))
      fail(SIVO_EINVAL, "fuse: null argument");
    fuse_device(*left->impl, targets, n_targets, *cam, points_device, n_points, th, match_device, dist_device, static_cast<cudaStream_t>(stream));
  });
}

int sivo_fuse(const sivo_orb_t* left, const sivo_keyframe_keys* targets, int n_targets, const sivo_fuse_camera* cam,
              const sivo_map_point* points, int n_points, float th, int* match, int* dist) {
  return guarded([&] {
    if (!left || !cam || (n_points > 0 && !points) || (n_targets > 0 && n_points > 0 && !match)) fail(SIVO_EINVAL, "fuse: null argument");
    fuse_host(*left->impl, targets, n_targets, *cam, points, n_points, th, match, dist, nullptr);
  });
}

int sivo_dbg_fuse(const sivo_orb_t* left, const sivo_keyframe_keys* targets, int n_targets, const sivo_fuse_camera* cam,
                  const sivo_map_point* points, int n_points, float th, int* match, int* dist, int* stage) {
  return guarded([&] {
    if (!left || !cam || (n_points > 0 && !points) || (n_targets > 0 && n_points > 0 && (!match || !dist || !stage)))
      fail(SIVO_EINVAL, "fuse: null argument");
    fuse_host(*left->impl, targets, n_targets, *cam, points, n_points, th, match, dist, stage);
  });
}

// ---------------------------------------------------------------------------------------- relocalisation PnP RANSAC
int sivo_pnp_create(const sivo_orb_t* left, int max_candidates, uint64_t seed, sivo_pnp_t** out) {
  return guarded([&] {
    if (!left || !out) fail(SIVO_EINVAL, "pnp_create: null argument");
    *out = nullptr;
    Pnp* impl = pnp_create(*left->impl, max_candidates, seed);
    *out = new sivo_pnp{impl};
  });
}

void sivo_pnp_destroy(sivo_pnp_t* h) {
  if (!h) return;
  pnp_destroy(h->impl);
  delete h;
}

int sivo_pnp_setup_device(sivo_pnp_t* h, const sivo_keypoint* kps_device, const int* keep_idx_device, const long long* n_keep_device,
                          const int* match_device, const long long* n_matches_device, const sivo_map_point* points_device,
                          int n_points, const uint32_t* kf_id, int n_kf, uint64_t frame_id, float fx, float fy, float cx, float cy,
                          void* stream) {
  return guarded([&] {
    if (!h || !kps_device || !n_keep_device || (n_kf > 0 && (!match_device || !n_matches_device)) || (n_points > 0 && !points_device))
      fail(SIVO_EINVAL, "pnp_setup: null argument");
    pnp_setup_device(*h->impl, kps_device, keep_idx_device, n_keep_device, match_device, n_matches_device, points_device, n_points, kf_id,
                     n_kf, frame_id, fx, fy, cx, cy, static_cast<cudaStream_t>(stream));
  });
}

int sivo_pnp_iterate_device(sivo_pnp_t* h, int n_iterations, const uint8_t* active, float* Tcw_device, int* has_pose_device,
                            int* no_more_device, int* inlier_match_device, int* n_inliers_device, void* stream) {
  return guarded([&] {
    if (!h || !Tcw_device || !has_pose_device || !no_more_device || !inlier_match_device || !n_inliers_device)
      fail(SIVO_EINVAL, "pnp_iterate: null argument");
    pnp_iterate_device(*h->impl, n_iterations, active, Tcw_device, has_pose_device, no_more_device, inlier_match_device, n_inliers_device,
                       static_cast<cudaStream_t>(stream));
  });
}

int sivo_dbg_pnp_state(const sivo_pnp_t* h, int* out, float* eps) {
  return guarded([&] {
    if (!h || !out) fail(SIVO_EINVAL, "pnp_state: null argument");
    pnp_state(*h->impl, out, eps);
  });
}

int sivo_dbg_pnp_compute_pose(int device, const float* p3d, const float* p2d, const float* max_err, int n, float fx, float fy, float cx,
                              float cy, double* alphas, uint32_t* mask, int* n_inliers, sivo_pnp_pose_debug* dbg) {
  return guarded([&] { pnp_compute_pose_debug(device, p3d, p2d, max_err, n, fx, fy, cx, cy, alphas, mask, n_inliers, dbg); });
}

int sivo_dbg_pnp_hypotheses(sivo_pnp_t* h, int k, int first, int n_hyp, int* draws, double* Rt, int* counts, uint32_t* masks) {
  return guarded([&] {
    if (!h || !draws || !Rt || !counts || !masks) fail(SIVO_EINVAL, "pnp_hypotheses: null argument");
    pnp_hypotheses(*h->impl, k, first, n_hyp, draws, Rt, counts, masks);
  });
}

int sivo_dbg_pnp_draws(int device, uint64_t seed, uint32_t kf_id, uint64_t frame_id, int first, int n_hyp, int N, int* out) {
  return guarded([&] { pnp_draws(device, seed, kf_id, frame_id, first, n_hyp, N, out); });
}

// ---------------------------------------------------------------------------------------- vocabulary and bag of words
int sivo_vocabulary_load_text(const char* path, int device, sivo_vocabulary_t** out) {
  return guarded([&] {
    if (!path || !out) fail(SIVO_EINVAL, "vocabulary_load_text: null argument");
    *out = nullptr;
    VocTree t;
    parse_vocabulary_text(path, t);
    auto* v = new Vocabulary(device, t.k, t.L, t.scoring, t.weighting, t.parent.data(), t.is_leaf.data(), t.desc.data(), t.weight.data(),
                             static_cast<int>(t.parent.size()));
    *out = new sivo_vocabulary{v};
  });
}

int sivo_vocabulary_create(int device, int k, int L, int scoring, int weighting, const int32_t* parent, const uint8_t* is_leaf,
                           const uint8_t* desc, const double* weight, int n_nodes, sivo_vocabulary_t** out) {
  return guarded([&] {
    if (!out || (n_nodes > 0 && (!parent || !is_leaf || !desc || !weight))) fail(SIVO_EINVAL, "vocabulary_create: null argument");
    *out = nullptr;
    auto* v = new Vocabulary(device, k, L, scoring, weighting, parent, is_leaf, desc, weight, n_nodes);
    *out = new sivo_vocabulary{v};
  });
}

int sivo_vocabulary_info(const sivo_vocabulary_t* voc, int* k, int* L, int* scoring, int* weighting, int* n_nodes, int* n_words) {
  return guarded([&] {
    if (!voc) fail(SIVO_EINVAL, "null handle");
    const Vocabulary& v = *voc->impl;
    if (k) *k = v.k;
    if (L) *L = v.L;
    if (scoring) *scoring = v.scoring;
    if (weighting) *weighting = v.weighting;
    if (n_nodes) *n_nodes = v.n_nodes;
    if (n_words) *n_words = v.n_words;
  });
}

void sivo_vocabulary_destroy(sivo_vocabulary_t* voc) {
  if (!voc) return;
  cudaSetDevice(voc->impl->device);
  delete voc->impl;
  delete voc;
}

int sivo_dbg_vocabulary_parse(const char* path, int* header, int* n_nodes, int32_t* parent, uint8_t* is_leaf, uint8_t* desc,
                              double* weight, int capacity) {
  return guarded([&] {
    if (!path || !header || !n_nodes) fail(SIVO_EINVAL, "vocabulary_parse: null argument");
    VocTree t;
    parse_vocabulary_text(path, t);
    const int n = static_cast<int>(t.parent.size());
    header[0] = t.k; header[1] = t.L; header[2] = t.scoring; header[3] = t.weighting;
    *n_nodes = n;
    if (capacity < n) fail(SIVO_ERANGE, "vocabulary_parse: %d nodes, room for %d", n, capacity);
    if (parent) std::copy(t.parent.begin(), t.parent.end(), parent);
    if (is_leaf) std::copy(t.is_leaf.begin(), t.is_leaf.end(), is_leaf);
    if (desc) std::copy(t.desc.begin(), t.desc.end(), desc);
    if (weight) std::copy(t.weight.begin(), t.weight.end(), weight);
  });
}

int sivo_compute_bow_device(const sivo_vocabulary_t* voc, const sivo_orb_t* left, const uint8_t* desc_device, const int* keep_idx_device,
                            const long long* n_keep_device, int levelsup, int* node_device, int* word_device, int* bow_word_device,
                            double* bow_weight_device, long long* bow_len_device, void* stream) {
  return guarded([&] {
    if (!voc || !left || !desc_device || !n_keep_device) fail(SIVO_EINVAL, "compute_bow: null argument");
    compute_bow_device(*voc->impl, *left->impl, desc_device, keep_idx_device, n_keep_device, levelsup, node_device, word_device,
                       bow_word_device, bow_weight_device, bow_len_device, static_cast<cudaStream_t>(stream));
  });
}

int sivo_compute_bow(const sivo_vocabulary_t* voc, const uint8_t* desc, int n, int levelsup, int* node, int* word, int* bow_word,
                     double* bow_weight, int* bow_len) {
  return guarded([&] {
    if (!voc) fail(SIVO_EINVAL, "compute_bow: null handle");
    compute_bow_host(*voc->impl, desc, n, levelsup, node, word, bow_word, bow_weight, bow_len);
  });
}

int sivo_search_by_bow_device(const sivo_orb_t* left, const sivo_keypoint* kps_device, const uint8_t* desc_device,
                              const int* keep_idx_device, const long long* n_keep_device, const int* node_device,
                              const sivo_keyframe_keys* keyframes, const int* const* kf_point_device, int n_kf, float nnratio,
                              int check_orientation, int* match_device, long long* n_matches_device, void* stream) {
  return guarded([&] {
    if (!left || !kps_device || !desc_device || !n_keep_device || !node_device || !match_device || !n_matches_device)
      fail(SIVO_EINVAL, "search_by_bow: null argument");
    search_by_bow_device(*left->impl, kps_device, desc_device, keep_idx_device, n_keep_device, node_device, keyframes, kf_point_device, n_kf,
                         nnratio, check_orientation, match_device, n_matches_device, static_cast<cudaStream_t>(stream));
  });
}

int sivo_search_by_bow(const sivo_orb_t* left, const sivo_keypoint* kps, const uint8_t* desc, const int* node, int n,
                       const sivo_keyframe_keys* keyframes, const int* const* kf_point, int n_kf, float nnratio, int check_orientation,
                       int* match, long long* n_matches) {
  return guarded([&] {
    if (!left) fail(SIVO_EINVAL, "search_by_bow: null handle");
    search_by_bow_host(*left->impl, kps, desc, node, n, keyframes, kf_point, n_kf, nnratio, check_orientation, match, n_matches);
  });
}

// ---------------------------------------------------------------------------------------- layer test hooks
namespace {
TensorView make_view(DevBuf& buf, int n, int c, int h, int w, int cs, DType dt) {
  TensorView v;
  v.n = n; v.c = c; v.h = h; v.w = w; v.cs = cs; v.dt = dt;
  buf.alloc(v.bytes());
  v.p = buf.p;
  return v;
}
void upload_nchw(const float* src, TensorView v) {
  size_t count = static_cast<size_t>(v.n) * v.c * v.h * v.w;
  DevBuf tmp(count * sizeof(float));
  SIVO_CUDA(cudaMemcpy(tmp.p, src, count * sizeof(float), cudaMemcpyHostToDevice));
  launch_nchw_to_act(tmp.as<float>(), v, nullptr);
  SIVO_CUDA(cudaDeviceSynchronize());
}
void download_nchw(TensorView v, float* dst) {
  size_t count = static_cast<size_t>(v.n) * v.c * v.h * v.w;
  DevBuf tmp(count * sizeof(float));
  launch_act_to_nchw(v, tmp.as<float>(), nullptr);
  SIVO_CUDA(cudaMemcpy(dst, tmp.p, count * sizeof(float), cudaMemcpyDeviceToHost));
}
}  // namespace

int sivo_dbg_pool(int device, const float* in, int n, int c, int h, int w, float* out, int* mask) {
  return guarded([&] {
    if (!in || n <= 0 || c <= 0 || (h & 1) || (w & 1)) fail(SIVO_EINVAL, "pool: bad arguments");
    SIVO_CUDA(cudaSetDevice(device));
    DevBuf bi, bo, bm(static_cast<size_t>(n) * c * (h / 2) * (w / 2)), bmi(static_cast<size_t>(n) * c * (h / 2) * (w / 2) * sizeof(int));
    TensorView vi = make_view(bi, n, c, h, w, c, DType::F32), vo = make_view(bo, n, c, h / 2, w / 2, c, DType::F32);
    upload_nchw(in, vi);
    launch_pool(vi, vo, bm.as<uint8_t>(), nullptr);
    if (out) download_nchw(vo, out);
    if (mask) {
      launch_mask_to_nchw(bm.as<uint8_t>(), n, c, h / 2, w / 2, bmi.as<int>(), nullptr);
      SIVO_CUDA(cudaMemcpy(mask, bmi.p, bmi.bytes, cudaMemcpyDeviceToHost));
    }
    SIVO_CUDA(cudaDeviceSynchronize());
  });
}

int sivo_dbg_unpool(int device, const float* in, const int* mask, int n, int c, int h, int w, float* out) {
  return guarded([&] {
    if (!in || !mask || !out) fail(SIVO_EINVAL, "unpool: null argument");
    SIVO_CUDA(cudaSetDevice(device));
    size_t cnt = static_cast<size_t>(n) * c * h * w;
    DevBuf bi, bo, bm(cnt), bmi(cnt * sizeof(int));
    TensorView vi = make_view(bi, n, c, h, w, c, DType::F32), vo = make_view(bo, n, c, h * 2, w * 2, c, DType::F32);
    upload_nchw(in, vi);
    SIVO_CUDA(cudaMemcpy(bmi.p, mask, cnt * sizeof(int), cudaMemcpyHostToDevice));
    launch_mask_from_nchw(bmi.as<int>(), n, c, h, w, bm.as<uint8_t>(), nullptr);
    launch_unpool(vi, bm.as<uint8_t>(), n, vo, nullptr);
    download_nchw(vo, out);
    SIVO_CUDA(cudaDeviceSynchronize());
  });
}

int sivo_dbg_lrn(int device, const float* in, int n, int c, int h, int w, int size, float alpha, float beta, float k, float* out) {
  return guarded([&] {
    if (!in || !out) fail(SIVO_EINVAL, "lrn: null argument");
    SIVO_CUDA(cudaSetDevice(device));
    DevBuf bi, bo;
    int cs = (c + 3) / 4 * 4;
    TensorView vi = make_view(bi, n, c, h, w, cs, DType::F32), vo = make_view(bo, n, c, h, w, cs, DType::F32);
    upload_nchw(in, vi);
    launch_lrn(vi, vo, size, alpha, beta, k, nullptr);
    download_nchw(vo, out);
    SIVO_CUDA(cudaDeviceSynchronize());
  });
}

int sivo_dbg_mc_reduce(int device, const float* logits, int T, int c, int h, int w, uint8_t* classes, double* confidence,
                       double* entropy) {
  return guarded([&] {
    if (!logits || T <= 0 || c <= 0) fail(SIVO_EINVAL, "mc_reduce: bad arguments");
    SIVO_CUDA(cudaSetDevice(device));
    DevBuf bl, bc(static_cast<size_t>(h) * w), bf(static_cast<size_t>(h) * w * 8), be(static_cast<size_t>(h) * w * 8);
    int cs = (c + 15) / 16 * 16;
    TensorView vl = make_view(bl, T, c, h, w, cs, DType::F32);
    upload_nchw(logits, vl);
    launch_mc_reduce(static_cast<const float*>(vl.p), T, c, cs, h * w, bc.as<uint8_t>(), bf.as<double>(), be.as<double>(), nullptr);
    SIVO_CUDA(cudaDeviceSynchronize());
    if (classes) SIVO_CUDA(cudaMemcpy(classes, bc.p, static_cast<size_t>(h) * w, cudaMemcpyDeviceToHost));
    if (confidence) SIVO_CUDA(cudaMemcpy(confidence, bf.p, static_cast<size_t>(h) * w * 8, cudaMemcpyDeviceToHost));
    if (entropy) SIVO_CUDA(cudaMemcpy(entropy, be.p, static_cast<size_t>(h) * w * 8, cudaMemcpyDeviceToHost));
  });
}

int sivo_dbg_mc_variance(int device, const float* logits, int T, int c, int h, int w, const uint8_t* classes, double* variance) {
  return guarded([&] {
    if (!logits || !classes || !variance || T < 2 || c <= 0 || h <= 0 || w <= 0) fail(SIVO_EINVAL, "mc_variance: bad arguments");
    SIVO_CUDA(cudaSetDevice(device));
    const size_t hw = static_cast<size_t>(h) * w;
    DevBuf bl, bc(hw), bv(hw * sizeof(double));
    int cs = (c + 15) / 16 * 16;  // the layout sivo_dbg_mc_reduce uses: C <= 16 takes the quad kernel, C > 16 the generic one
    TensorView vl = make_view(bl, T, c, h, w, cs, DType::F32);
    upload_nchw(logits, vl);
    SIVO_CUDA(cudaMemcpy(bc.p, classes, hw, cudaMemcpyHostToDevice));
    launch_mc_variance(static_cast<const float*>(vl.p), T, c, cs, static_cast<int>(hw), bc.as<uint8_t>(), bv.as<double>(), nullptr);
    SIVO_CUDA(cudaDeviceSynchronize());
    SIVO_CUDA(cudaMemcpy(variance, bv.p, hw * sizeof(double), cudaMemcpyDeviceToHost));
  });
}

int sivo_dbg_dropout_mask(int device, uint64_t seed, uint64_t frame, int layer, int T, int c, int h, int w, uint8_t* keep) {
  return guarded([&] {
    if (!keep) fail(SIVO_EINVAL, "dropout_mask: null output");
    SIVO_CUDA(cudaSetDevice(device));
    size_t cnt = static_cast<size_t>(T) * c * h * w;
    DevBuf bk(cnt), bf(8);
    SIVO_CUDA(cudaMemcpy(bf.p, &frame, 8, cudaMemcpyHostToDevice));
    launch_dropout_bits(seed, bf.as<uint64_t>(), layer, T, c, h, w, bk.as<uint8_t>(), nullptr);
    SIVO_CUDA(cudaMemcpy(keep, bk.p, cnt, cudaMemcpyDeviceToHost));
  });
}

int sivo_dbg_conv(int device, int engine, int precision, const float* in, int n, int cin, int h, int w, const float* weight,
                  const float* bias, const float* bn_scale, const float* bn_shift, int cout, int k, int pad, int relu,
                  float* out) {
  return guarded([&] {
    if (!in || !weight || !out) fail(SIVO_EINVAL, "conv: null argument");
    if (pad != (k - 1) / 2) fail(SIVO_EINVAL, "conv: only 'same' padding");
    SIVO_CUDA(cudaSetDevice(device));
    DType dt = precision == SIVO_PRECISION_FP32 ? DType::F32 : DType::F16;
    int cs_in = cin < 8 ? 4 : cin;
    if (cin >= 8 && cin % 8) fail(SIVO_EINVAL, "conv: cin must be 3/4 or a multiple of 8");
    DevBuf bi, bo;
    TensorView vi = make_view(bi, n, cin, h, w, cs_in, dt);
    int cs_out = (cout % 8) ? (cout + 15) / 16 * 16 : cout;
    DType odt = (cout % 8) ? DType::F32 : dt;
    TensorView vo = make_view(bo, n, cout, h, w, cs_out, odt);
    upload_nchw(in, vi);
    Op op;  // the network's convolution op, prepared and launched as SegNet does
    op.kind = Op::Conv;
    op.layer = "dbg_conv";
    op.k = k; op.pad = pad; op.cin = cin; op.cout = cout; op.cin_p = cs_in; op.cout_p = (cout + 63) / 64 * 64;
    op.relu = relu != 0;
    if (engine == SIVO_ENGINE_TCGEN05 && dt == DType::F32) {  // split-operand fp32 mode
      op.split = op.use_tc = true;
      if (cin % 64 || !conv_tc_supported(op, split_view(vi), vo))
        fail(SIVO_EINVAL, "conv: shape not supported by the split-operand tcgen05 mode");
    } else if (engine == SIVO_ENGINE_TCGEN05) {
      op.use_tc = true;
      if (dt != DType::F16 || !conv_tc_supported(op, vi, vo)) fail(SIVO_EINVAL, "conv: shape not supported by the tcgen05 engine");
    }
    prepare_conv(op, dt, weight, bias, bn_scale, bn_shift, vi, vo);
    launch_conv(op, vi, vo, nullptr);
    SIVO_CUDA(cudaDeviceSynchronize());
    download_nchw(vo, out);
    SIVO_CUDA(cudaDeviceSynchronize());
  });
}

int sivo_dbg_conv_unpooled(int device, const float* pooled, const int* mask, int n, int mask_n, int h, int w, const float* weight,
                           const float* bias, const float* bn_scale, const float* bn_shift, int cout, int k, float* out) {
  return guarded([&] {
    if (!pooled || !mask || !weight || !out) fail(SIVO_EINVAL, "conv_unpooled: null argument");
    if (n < 1 || mask_n < 1 || mask_n > n || h < 1 || w < 1 || cout < 1 || cout > 16 || k != 7)
      fail(SIVO_EINVAL, "conv_unpooled: needs n, h, w >= 1, 1 <= mask_n <= n, 1 <= cout <= 16 and k = 7");
    SIVO_CUDA(cudaSetDevice(device));
    const size_t mask_cnt = static_cast<size_t>(mask_n) * 64 * h * w;
    DevBuf bp, bo, bm(mask_cnt), bmi(mask_cnt * sizeof(int));
    TensorView vp = make_view(bp, n, 64, h, w, 64, DType::F16);
    TensorView vo = make_view(bo, n, cout, 2 * h, 2 * w, 16, DType::F32);
    upload_nchw(pooled, vp);
    SIVO_CUDA(cudaMemcpy(bmi.p, mask, mask_cnt * sizeof(int), cudaMemcpyHostToDevice));
    launch_mask_from_nchw(bmi.as<int>(), mask_n, 64, h, w, bm.as<uint8_t>(), nullptr);
    Op op;
    op.kind = Op::Conv;
    op.layer = "dbg_conv_unpooled";
    op.k = k; op.pad = (k - 1) / 2; op.cin = op.cin_p = 64; op.cout = cout; op.cout_p = 64;
    op.use_tc = true;
    TensorView vu = vp;  // the unpooled input's shape: the plan is made for it, and then reads the pooled tensor instead
    vu.h = 2 * h;
    vu.w = 2 * w;
    if (!conv_tc_supported(op, vu, vo)) fail(SIVO_EINVAL, "conv_unpooled: shape not supported by the tensor-core kernel");
    prepare_conv(op, DType::F16, weight, bias, bn_scale, bn_shift, vu, vo);
    conv_tc_set_unpool_input(*op.tc, vp.p, bm.as<uint8_t>(), mask_n, h, w);
    launch_conv(op, vu, vo, nullptr);
    SIVO_CUDA(cudaDeviceSynchronize());
    download_nchw(vo, out);
    SIVO_CUDA(cudaDeviceSynchronize());
  });
}

int sivo_dbg_conv64_unpooled(int device, const float* pooled, const int* mask, int n, int mask_n, int h, int w, const float* weight,
                             const float* bias, int drop_layer, uint64_t seed, uint64_t frame, int unpool_on_load, float* out) {
  return guarded([&] {
    if (!pooled || !mask || !weight || !out) fail(SIVO_EINVAL, "conv64_unpooled: null argument");
    if (n < 1 || mask_n < 1 || mask_n > n || h < 1 || w < 1) fail(SIVO_EINVAL, "conv64_unpooled: needs n, h, w >= 1 and 1 <= mask_n <= n");
    SIVO_CUDA(cudaSetDevice(device));
    const size_t mask_cnt = static_cast<size_t>(mask_n) * 64 * h * w;
    DevBuf bp, bu, bo, bm(mask_cnt), bmi(mask_cnt * sizeof(int)), bf(sizeof(uint64_t));
    TensorView vp = make_view(bp, n, 64, h, w, 64, DType::F16);
    TensorView vu = make_view(bu, n, 64, 2 * h, 2 * w, 64, DType::F16);
    TensorView vo = make_view(bo, n, 64, 2 * h, 2 * w, 64, DType::F16);
    upload_nchw(pooled, vp);
    SIVO_CUDA(cudaMemcpy(bmi.p, mask, mask_cnt * sizeof(int), cudaMemcpyHostToDevice));
    SIVO_CUDA(cudaMemcpy(bf.p, &frame, sizeof(uint64_t), cudaMemcpyHostToDevice));
    launch_mask_from_nchw(bmi.as<int>(), mask_n, 64, h, w, bm.as<uint8_t>(), nullptr);
    Op op;
    op.kind = Op::Conv;
    op.layer = "dbg_conv64_unpooled";
    op.k = 7; op.pad = 3; op.cin = op.cin_p = 64; op.cout = op.cout_p = 64;
    op.use_tc = true;
    if (!conv_tc_supported(op, vu, vo)) fail(SIVO_EINVAL, "conv64_unpooled: shape not supported by the tensor-core kernel");
    prepare_conv(op, DType::F16, weight, bias, nullptr, nullptr, vu, vo);
    if (drop_layer >= 0) conv_tc_set_dropout(*op.tc, seed, bf.as<uint64_t>(), drop_layer, 2.f, 0);
    if (unpool_on_load) conv_tc_set_unpool_input(*op.tc, vp.p, bm.as<uint8_t>(), mask_n, h, w);
    else launch_unpool(vp, bm.as<uint8_t>(), mask_n, vu, nullptr);
    launch_conv(op, vu, vo, nullptr);
    SIVO_CUDA(cudaDeviceSynchronize());
    download_nchw(vo, out);
    SIVO_CUDA(cudaDeviceSynchronize());
  });
}

}  // extern "C"
