/* sivo_b200 -- C ABI of the H100-native (sm_90a) SIVO perception front-end (libsivo_b200.so).
 *
 * The reference has no FFI on this path: the "plugin API" is two C++ classes.  The shim classes in
 * integration/ keep their public signatures and forward to the entry points below, so src/sivo.cc,
 * src/orbslam/System.cc, Tracking.cc and Frame.cc compile unchanged (see INTEGRATION.md).
 *
 *   sivo_segnet_*   replaces  SIVO::BayesianSegNet            include/bayesian_segnet/bayesian_segnet.hpp:108-170
 *                             ctor                             src/bayesian_segnet/bayesian_segnet.cpp:46-78
 *                             segmentImage                     src/bayesian_segnet/bayesian_segnet.cpp:299-318
 *                             getInputGeometry                 include/bayesian_segnet/bayesian_segnet.hpp:139
 *                             computeVariance                  src/bayesian_segnet/bayesian_segnet.cpp:205-260
 *   sivo_orb_*      replaces  SIVO::ORBextractor              include/orbslam/ORBextractor.h:46-125
 *                             ctor                             src/orbslam/ORBextractor.cc:412-475
 *                             operator()                       src/orbslam/ORBextractor.cc:1019-1083
 *                             mvImagePyramid (public member)   include/orbslam/ORBextractor.h:90
 *   sivo_stereo_*   replaces  the Hamming stage of Frame::ComputeStereoMatches   src/orbslam/Frame.cc:444-533
 *                             ORBmatcher::DescriptorDistance   src/orbslam/ORBmatcher.cc:1582-1596
 *
 * Conventions: every function returns 0 on success or a negative SIVO_E* code and never throws or aborts
 * across the boundary; sivo_last_error() returns a thread-local message for the last failure on the
 * calling thread.  Pointers are plain host pointers unless the name says `_device`.  Handles are
 * independent: two sivo_orb_t may be driven concurrently from two threads (Frame.cc:126-129); one handle
 * must not be used from two threads at once.  A `_device` call's scratch is its own: allocated and freed on its `stream`
 * (stream-ordered, no host synchronisation), never on an extractor.  So calls on different streams share only the buffers they
 * are given, and a call's inputs (e.g. the keypoints the next sivo_orb_enqueue_device into the same buffers rewrites) must not be
 * rewritten until it has run.
 */
#ifndef SIVO_B200_H_
#define SIVO_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SIVO_OK 0
#define SIVO_EINVAL (-22)   /* bad argument; the shim rethrows std::invalid_argument where the reference does */
#define SIVO_ENOENT (-2)    /* prototxt / caffemodel not readable */
#define SIVO_EFORMAT (-74)  /* prototxt / caffemodel malformed, unsupported layer, LFS stub, shape mismatch */
#define SIVO_ECUDA (-5)     /* CUDA runtime / driver error (message has the cudaError string) */
#define SIVO_ENOMEM (-12)
#define SIVO_ERANGE (-34)   /* output capacity too small */

typedef struct sivo_segnet sivo_segnet_t;
typedef struct sivo_orb sivo_orb_t;

/* bit-compatible with cv::KeyPoint (pt.x, pt.y, size, angle, response, octave, class_id) */
typedef struct sivo_keypoint {
  float x, y, size, angle, response;
  int32_t octave, class_id;
} sivo_keypoint;

/* precision of the convolution operands (accumulation is always fp32, the MC reduction fp64) */
enum { SIVO_PRECISION_FP16 = 0, SIVO_PRECISION_FP32 = 1 };
/* convolution engine */
enum { SIVO_ENGINE_AUTO = 0, SIVO_ENGINE_SIMT = 1, SIVO_ENGINE_TCGEN05 = 2 };

typedef struct sivo_segnet_options {
  int32_t device;      /* CUDA device ordinal */
  int32_t T;           /* MC samples; 0 = take the prototxt's first input dim */
  uint64_t seed;       /* dropout seed (oracle/philox.py spells out the mask rule) */
  int32_t precision;   /* SIVO_PRECISION_* */
  int32_t engine;      /* SIVO_ENGINE_* */
  int32_t keep_blobs;  /* 1 = keep every intermediate blob for sivo_segnet_blob (tests); disables fusion */
  int32_t reserved;
} sivo_segnet_options;

/* ---- Bayesian SegNet -------------------------------------------------------------------------- */
/* Fails with SIVO_EINVAL for NULL/empty paths, input C != 3, T <= 1 (bayesian_segnet.cpp:65-70,80-89). */
int sivo_segnet_create(const char* prototxt, const char* caffemodel, int device, uint64_t seed,
                       sivo_segnet_t** out);
int sivo_segnet_create_ex(const char* prototxt, const char* caffemodel, const sivo_segnet_options* opt,
                          sivo_segnet_t** out);
int sivo_segnet_geometry(const sivo_segnet_t* h, int* width, int* height, int* T, int* n_classes);
/* Dropout masks are keyed by (seed, frame, layer, sample, element); frame auto-increments per run. */
int sivo_segnet_set_frame(sivo_segnet_t* h, uint64_t frame);
/* segmentImage: bgr is rows x cols x 3 u8 with `stride` bytes per row; larger images are centre-cropped
 * (resizeImage, bayesian_segnet.cpp:142-162), smaller ones are SIVO_EINVAL.  Outputs are row-major
 * height x width (MatXu / MatXd layout, bayesian_segnet.hpp:46-50); any of them may be NULL. */
int sivo_segnet_run(sivo_segnet_t* h, const uint8_t* bgr, int rows, int cols, size_t stride,
                    uint8_t* classes, double* confidence, double* entropy);
/* Same with device-resident buffers (already cropped height x width x 3, tightly packed) on `stream`
 * (a cudaStream_t; NULL = the handle's own stream).  No host synchronisation. */
int sivo_segnet_run_device(sivo_segnet_t* h, const uint8_t* bgr_device, uint8_t* classes_device,
                           double* confidence_device, double* entropy_device, void* stream);
/* Multi-GPU callers share a packed per-frame record (SURVEY 8e): after this call every sivo_segnet_run additionally leaves the
 * classes (u8) and single-precision copies of the confidence / entropy maps at these DEVICE addresses, complete when it returns,
 * so the record's maps never travel host -> device.  All NULL switches it off. */
int sivo_segnet_set_record_outputs(sivo_segnet_t* h, uint8_t* classes_device, float* confidence_f32_device, float* entropy_f32_device);
/* The same with additional single-precision copies of the two maps (any output may be NULL): what the packed per-frame record
 * of the multi-GPU path carries (SURVEY 8e: classes u8 + entropy f32 + confidence f32), written straight into it by the MC
 * reduction; the double maps stay the operator's outputs (bayesian_segnet.cpp:192-203, 262-276 compute in double). */
int sivo_segnet_run_device_maps(sivo_segnet_t* h, const uint8_t* bgr_device, uint8_t* classes_device, double* confidence_device,
                                double* entropy_device, float* confidence_f32_device, float* entropy_f32_device, void* stream);
/* ---- latency mode (SURVEY 8e): one frame's Monte-Carlo samples split across GPUs ------------------------------------
 * A shard handle owns the samples [sample_begin, sample_begin + sample_count) of a frame of opt->T samples (0 = the prototxt's
 * batch): it runs the sample-invariant prefix once and the rest of the net for its own samples only, and sample n of the shard
 * draws exactly the dropout masks sample sample_begin + n draws in a whole-frame handle with the same seed and frame counter.
 * Each rank sums its samples' softmax (sivo_segnet_run_partial_device), the sums are added across ranks (e.g. one reduce),
 * and one rank turns the total into the operator's maps (sivo_segnet_finalize_device).  A handle from sivo_segnet_create_ex is
 * the shard [0, T).  SIVO_EINVAL for sample_begin < 0, sample_count < 1 or sample_begin + sample_count > T, and for T <= 1 as
 * in sivo_segnet_create.  sivo_segnet_run, _run_device and _run_device_maps refuse a shard that owns fewer than T samples
 * (SIVO_EINVAL).  The frame counter advances per sivo_segnet_run_partial_device exactly as per sivo_segnet_run_device, so
 * shards created alike and pinned with sivo_segnet_set_frame stay in lockstep. */
int sivo_segnet_create_shard(const char* prototxt, const char* caffemodel, const sivo_segnet_options* opt, int sample_begin,
                             int sample_count, sivo_segnet_t** out);
/* The handle's sample range and the frame's sample count T (the mean divides by T); any output may be NULL. */
int sivo_segnet_samples(const sivo_segnet_t* h, int* sample_begin, int* sample_count, int* T_total);
/* bgr_device as in sivo_segnet_run_device.  sum_device: height*width x 16 doubles, pixel-major, overwritten with the sum over
 * the shard's samples of the per-sample softmax (the per-sample arithmetic of the one-pass reduction; channels >= n_classes
 * are 0).  On `stream` (NULL = the handle's own), no host synchronisation.  SIVO_EINVAL for a NULL image or sum; SIVO_EFORMAT
 * if the net has more than 16 classes. */
int sivo_segnet_run_partial_device(sivo_segnet_t* h, const uint8_t* bgr_device, double* sum_device, void* stream);
/* sum_device: the sum over ALL T samples of the frame (e.g. the shards' sums after a reduction over ranks), layout as above.
 * Writes what sivo_segnet_run_device_maps writes, any output may be NULL; the shard [0, T) followed by this call gives the same
 * bits as sivo_segnet_run_device_maps.  The maps become the ones sivo_segnet_semantic_keys reads.  Does not touch the frame
 * counter.  On `stream` (NULL = the handle's own), no host synchronisation; SIVO_EINVAL for a NULL sum. */
int sivo_segnet_finalize_device(sivo_segnet_t* h, const double* sum_device, uint8_t* classes_device, double* confidence_device,
                                double* entropy_device, float* confidence_f32_device, float* entropy_f32_device, void* stream);
/* ---- Monte-Carlo variance (BayesianSegNet::computeVariance, bayesian_segnet.cpp:205-260) ------------------------------
 * Per pixel, with c = classes[row * width + col] (normally the class map the same frame's run returned) and p_t the softmax
 * probability of class c in sample t of the LAST FRAME RUN ON THE HANDLE: avg = sum_t p_t / T and variance = sum_t (p_t - avg)^2
 * / (T - 1), the sample variance, summed in double in sample order.  Two rules the reference leaves open: a class >= n_classes
 * (e.g. VOID = 255) gives 0, and p_t is computed with the per-sample arithmetic of the reduction the handle runs, so for the
 * argmax class avg is the mean `confidence` reports.  The samples never leave the device, so only these calls can compute it.
 * They do not touch the frame counter.  SIVO_EINVAL for a NULL buffer or a handle that has not run a frame yet.
 *
 * Host form: classes (u8) and variance (double) are row-major height x width host buffers; returns when done.  SIVO_EINVAL on
 * a latency-mode shard owning fewer than T samples. */
int sivo_segnet_variance(sivo_segnet_t* h, const uint8_t* classes, double* variance);
/* The same with device buffers on `stream` (NULL = the handle's own), no host synchronisation.  The call must be ordered after
 * the run whose samples it reads (the same stream, or a stream that waits on it) and before the handle's next run, which
 * overwrites them. */
int sivo_segnet_variance_device(sivo_segnet_t* h, const uint8_t* classes_device, double* variance_device, void* stream);
/* Latency mode: moments_device (height*width x 2 doubles, pixel-major) = (sum p_t, sum p_t^2) of class c over this shard's
 * samples of its last sivo_segnet_run_partial_device ((0, 0) where c >= n_classes); ordered as above.  SIVO_EFORMAT if the
 * net's logits do not have the 16-channel layout (more than 16 classes), as sivo_segnet_run_partial_device. */
int sivo_segnet_variance_partial_device(sivo_segnet_t* h, const uint8_t* classes_device, double* moments_device, void* stream);
/* moments_device: the moments summed over ALL T samples of the frame (e.g. reduced over the ranks).  variance_device =
 * max(0, (S2 - S1^2 / T) / (T - 1)); agrees with the two-pass form to rounding (about 1e-16 for probabilities). */
int sivo_segnet_variance_finalize_device(sivo_segnet_t* h, const double* moments_device, double* variance_device, void* stream);
/* Test hook: copies blob `name` (any top in the prototxt; needs keep_blobs) to `out` as float NCHW.
 * `*n`, `*c`, `*hh`, `*ww` receive its shape; `out` may be NULL to query the shape only. */
int sivo_segnet_blob(sivo_segnet_t* h, const char* name, float* out, size_t cap, int* n, int* c, int* hh,
                     int* ww);
/* Enables per-op CUDA-event timing (adds a host sync per run); off by default. */
/* Frame::SelectSemanticKeys (Frame.cc:177-203) plus the per-keypoint reads of the three maps that Tracking / LocalMapping
 * do later (Tracking.cc:487,538; LocalMapping.cc:483-485), evaluated on the device-resident maps of the last
 * sivo_segnet_run / _run_device -- so a caller that only needs per-keypoint values can pass NULL maps to sivo_segnet_run
 * and skip the 6.1 MB read-back.  For keypoint i: (row, col) = ((int) y, (int) x); kp_class/kp_conf/kp_entropy[i] = the map
 * values there (class 255, 0, 0 and never kept if outside the maps, or if x or y is not finite -- the reference would read out of
 * bounds or convert a NaN to int; the test is made in float, before the conversion).
 * keep_idx[0..*n_keep) = indices with class <= max_static_class (Classes::TERRAIN = 8 in the reference), ascending, i.e. the
 * order mvKeysSemantic / mDescriptorsSemantic are built in.  Any output pointer may be NULL. */
int sivo_segnet_semantic_keys(sivo_segnet_t* h, const sivo_keypoint* kps, int n, int max_static_class, uint8_t* kp_class,
                              double* kp_conf, double* kp_entropy, int* keep_idx, int* n_keep);
/* The same selection for a device-resident pipeline: keypoints, count and every output are DEVICE buffers, e.g. what
 * sivo_orb_enqueue_device leaves (kps_device, and its int64 *count_device, read on the device).  The maps are those of the
 * handle's last run (sivo_segnet_run / _run_device / _run_device_maps / _finalize_device) as they stand when the call is made.
 * cap = capacity of the caller's buffers (kp_class / kp_conf / kp_entropy / keep_idx hold cap entries each; sivo_orb_capacity
 * suffices for an extractor's output).  If *count_device > cap (or < 0) nothing is written except *n_keep_device = -1.  Otherwise
 * the per-key values and keep_idx[0 .. *n_keep_device) equal the host form's bit for bit (keep_idx ascending).  Any output may
 * be NULL.  Runs on `stream` (NULL = the stream of the handle's last run) with no host synchronisation and no host staging; the
 * stream must be ordered after the run that wrote the maps and after the producer of the keypoints (e.g. sivo_orb_stream_wait),
 * and before the next run overwrites the maps.  SIVO_EINVAL for a NULL handle, keypoint or count pointer, a negative cap, or a
 * handle with no maps on the device yet. */
int sivo_segnet_semantic_keys_device(sivo_segnet_t* h, const sivo_keypoint* kps_device, const long long* count_device, int cap,
                                     int max_static_class, uint8_t* kp_class_device, double* kp_conf_device,
                                     double* kp_entropy_device, int* keep_idx_device, long long* n_keep_device, void* stream);
int sivo_segnet_set_profiling(sivo_segnet_t* h, int on);
/* Per-stage device times (ms) of the last run: conv, other layers, MC reduction, total; counts kernels. */
int sivo_segnet_last_timing(const sivo_segnet_t* h, float* conv_ms, float* other_ms, float* reduce_ms,
                            float* total_ms, int* launches);
int sivo_segnet_flops(const sivo_segnet_t* h, double* conv_flops_dedup, double* conv_flops_naive);
/* One launch of the op list (index < 0: only `*n_ops`): layer name(s) it covers, its time in the last profiled run
 * (ms, CUDA events on the launching stream) and its algorithmic convolution flops (0 for non-convolution launches). */
int sivo_segnet_op_timing(const sivo_segnet_t* h, int index, char* name, size_t cap, float* ms, double* flops,
                          int* n_ops);
/* Multiply-add work a launch EXECUTES on the tensor / CUDA cores, as flops (2 x MACs).  Equals the algorithmic figure of
 * sivo_segnet_op_timing except where the library changes the operation count: the composed conv_decode1 x classifier layer
 * (one 64 -> 16 7x7 convolution instead of 64 -> 64 followed by 64 -> 15: 0.25x) and the split-operand fp32 mode (3x). */
int sivo_segnet_op_flops_executed(const sivo_segnet_t* h, int index, double* flops);
void sivo_segnet_destroy(sivo_segnet_t* h);

/* ---- ORB extractor ---------------------------------------------------------------------------- */
int sivo_orb_create(int nfeatures, float scale_factor, int nlevels, int ini_th_fast, int min_th_fast,
                    int device, sivo_orb_t** out);
/* Scale tables, each `nlevels` floats (GetScaleFactors & co, ORBextractor.h:66-88); any may be NULL. */
int sivo_orb_tables(const sivo_orb_t* h, float* scale, float* inv_scale, float* sigma2, float* inv_sigma2,
                    int* features_per_level);
/* operator(): gray is rows x cols u8.  Writes up to `cap` keypoints (level-major order) and cap x 32
 * descriptor bytes, *n = count (SIVO_ERANGE if cap is too small; nfeatures + 3*nlevels always suffices).
 * If pyramid_levels != NULL it must hold nlevels host pointers to buffers of
 * (level_h + 38) * pyramid_strides[l] bytes which receive the bordered level images, i.e. what
 * mvImagePyramid[l] is a (19,19)-offset ROI of (query sizes with sivo_orb_level_size). */
int sivo_orb_run(sivo_orb_t* h, const uint8_t* gray, int rows, int cols, size_t stride, sivo_keypoint* kps,
                 int cap, int* n, uint8_t* desc32, uint8_t* const* pyramid_levels,
                 const size_t* pyramid_strides);
/* Same operator with the gray image already resident in device memory (`pitch` bytes per row); the
 * candidate / selection round trip through the host quad tree stays inside the call. */
int sivo_orb_run_device_input(sivo_orb_t* h, const uint8_t* gray_device, int rows, int cols, size_t pitch,
                              sivo_keypoint* kps, int cap, int* n, uint8_t* desc32);
/* Fully asynchronous operator for device-resident pipelines (frame sharding across GPUs, CUDA-graph style callers): enqueues
 * pyramid -> FAST -> cells -> device quad tree -> blur -> rBRIEF on the handle's own stream and returns without synchronising.
 * kps_device needs room for sivo_orb_capacity(h) records, desc32_device for 32 bytes each; *count_device (int64) receives the
 * keypoint count, or -1 if a pyramid level exceeded the device tree's capacity (more than 8,192 FAST candidates, more than 16
 * initial quad-tree nodes, or more nodes than its shared memory holds): the records are then not valid, and the device forms of the
 * Frame tail that read the count write their own -1 and nothing else.  sivo_orb_stream_wait makes another stream wait for the
 * enqueued work; sivo_orb_device_status (synchronises) returns the mask of those levels (sivo_orb_run extracts such inputs). */
int sivo_orb_enqueue_device(sivo_orb_t* h, const uint8_t* gray_device, int rows, int cols, size_t pitch, sivo_keypoint* kps_device,
                            uint8_t* desc32_device, long long* count_device);
int sivo_orb_stream_wait(sivo_orb_t* h, void* consumer_cuda_stream);
/* The reverse edge: the handle's stream waits for everything enqueued on `producer_cuda_stream` so far (e.g. the collective
 * that still reads the buffers the next sivo_orb_enqueue_device will overwrite). */
int sivo_orb_wait_for_stream(sivo_orb_t* h, void* producer_cuda_stream);
/* The same edge for one recorded event (a cudaEvent_t): the handle's stream waits for exactly that point of another stream. */
int sivo_orb_wait_event(sivo_orb_t* h, void* cuda_event);
int sivo_orb_device_status(sivo_orb_t* h, int* level_mask);
int sivo_orb_capacity(const sivo_orb_t* h, int* max_keypoints);
int sivo_orb_has_device_tree(const sivo_orb_t* h, int* yes);
int sivo_orb_level_size(const sivo_orb_t* h, int rows, int cols, int level, int* level_w, int* level_h);
/* Test hook: FAST candidates of the last run before the quad tree, per level (x, y relative to the
 * (16,16) border origin as in ComputeKeyPointsOctTree, response). */
int sivo_orb_candidates(const sivo_orb_t* h, int level, int* xs, int* ys, int* resp, int cap, int* n);
int sivo_orb_last_timing(const sivo_orb_t* h, float* device_ms, float* host_tree_ms, int* launches);
void sivo_orb_destroy(sivo_orb_t* h);

/* Host-only DistributeOctTree (ORBextractor.cc:544-750), exported so that the shim, the library and the
 * tests share one implementation of the documented tie rule.  Returns the number of kept indices. */
int sivo_orb_distribute(const float* xs, const float* ys, const float* resp, int n, int min_x, int max_x,
                        int min_y, int max_y, int n_target, int* keep, int cap);

/* Test hook: the same distribution on the DEVICE quad tree (orb_tree.cu), integer key coordinates < 4096 and responses < 256
 * as the FAST stage produces them.  Writes the kept keys' (x, y, response) in list order; returns their count, or
 * SIVO_ERANGE if the input exceeds the device tree's capacity. */
int sivo_dbg_orb_distribute_device(int device, const int* xs, const int* ys, const int* resp, int n, int min_x, int max_x,
                                   int min_y, int max_y, int n_target, int* out_x, int* out_y, int* out_resp, int cap);

/* ---- stereo Hamming stage (next-row 1) -------------------------------------------------------- */
/* For each left keypoint: best right candidate in its row band (rows vL +- 2*scale[octave]), octave
 * within +-1, uR in [uL - max_d, uL - min_d], minimal DescriptorDistance; best_idx = -1 if none.
 * Mirrors Frame.cc:452-533 up to (not including) the SAD refinement.  A left key with a non-finite x or y, or with (int) y outside
 * [0, rows), has no candidate; a right key with a non-finite x or y is never a candidate (sivo_stereo_match's rule).
 * SIVO_EINVAL for n_right >= 2^20 (the search packs the right index into 20 bits). */
int sivo_stereo_hamming(int device, const sivo_keypoint* left, const uint8_t* desc_left, int n_left,
                        const sivo_keypoint* right, const uint8_t* desc_right, int n_right,
                        const float* scale_factors, int nlevels, int rows, float min_d, float max_d,
                        int* best_idx, int* best_dist);

/* Test hook: the median-based outlier cut of sivo_stereo_match alone.  sad[i] < 0 marks key i unmatched; with m matched keys the
 * median is the SAD of rank m / 2 in ascending order, and every matched key with (float) sad >= 1.5f * 1.4f * median gets
 * u[i] = z[i] = -1 (u and z are read and written in place, n entries each). */
int sivo_dbg_stereo_median_cut(int device, const int* sad, int n, float* u, float* z);

/* The whole of Frame::ComputeStereoMatches (Frame.cc:444-629): Hamming search, 11x11 SAD slide (+-5 px) on the keypoint's
 * pyramid level, parabola sub-pixel fit, disparity gate [0, mbf/mb), median-based outlier cut.  Uses the device-resident
 * pyramids of the last sivo_orb_run of `left` / `right` (so mvImagePyramid need not travel to the host for it).
 * u_right / depth: n_left floats each = mvRight / mvDepth (-1 where unmatched).
 * Rule where the reference throws or is undefined (it changes nothing for keys an extractor produces): a left key stays unmatched,
 * and no SAD of it enters the median, if its x or y is not finite, if (int) y is outside [0, rows), if its 11 x 11 window at its
 * octave leaves that level's image (rows sv_l +- 5, columns su_l +- 5), or if the right slide does (rows sv_l +- 5, columns
 * su_r0 - 10 .. su_r0 + 10); a right key with a non-finite x or y is never a candidate.  Every test is made in float, before any
 * conversion to int; the reference's own endu >= cols test stays as written.  SIVO_EINVAL, before anything is launched or
 * written, if the two extractors' last runs have different level tables (image size or scale factor), and for n_right >= 2^20. */
int sivo_stereo_match(const sivo_orb_t* left, const sivo_orb_t* right, const sivo_keypoint* kp_left, const uint8_t* desc_left,
                      int n_left, const sivo_keypoint* kp_right, const uint8_t* desc_right, int n_right, float mb, float mbf,
                      float* u_right, float* depth);
/* The same on device-resident inputs and outputs, e.g. the buffers sivo_orb_enqueue_device filled for `left` / `right`.
 * Output j (u_right_device[j], depth_device[j]) belongs to left keypoint keep_idx_device[j] for j < *n_left_device, or to left
 * keypoint j when keep_idx_device is NULL: pass sivo_segnet_semantic_keys_device's keep_idx / n_keep to match mvKeysSemantic.
 * The values equal sivo_stereo_match's on the same keypoints gathered on the host (-1 where unmatched), median cut included.
 * Counts (int64) are read on the device and clamped to the extractors' capacities; a negative *n_left_device (the -1 of
 * sivo_segnet_semantic_keys_device) writes nothing.  The output buffers need sivo_orb_capacity(left) floats.  Keypoints whose
 * octave is outside [0, nlevels) are left unmatched.
 * Ordering: the call makes `stream` (NULL = the left extractor's stream) wait for everything enqueued so far on both extractors'
 * streams, so no manual wait is needed after sivo_orb_enqueue_device; keep_idx / n_keep must be ordered before it on `stream`.  The
 * call reads both pyramids, so the next sivo_orb_enqueue_device on either extractor must be ordered after it
 * (sivo_orb_wait_for_stream(extractor, stream)).  No host synchronisation.  SIVO_EINVAL for NULL handles or buffers (keep_idx_device may be NULL), extractors
 * that have not run, extractors on different devices, with different nlevels or different level tables, mb / mbf <= 0, and a right
 * extractor whose sivo_orb_capacity is >= 2^20; nothing is enqueued then.  Keys follow sivo_stereo_match's rule. */
int sivo_stereo_match_device(sivo_orb_t* left, sivo_orb_t* right, const sivo_keypoint* kp_left_device, const uint8_t* desc_left_device,
                             const int* keep_idx_device, const long long* n_left_device, const sivo_keypoint* kp_right_device,
                             const uint8_t* desc_right_device, const long long* n_right_device, float mb, float mbf,
                             float* u_right_device, float* depth_device, void* stream);

/* ---- SIVO's information-based map-point selection (Tracking::StereoInitialization, Tracking.cc:470-520, threshold 0;
 * Tracking::CreateNewKeyFrame, Tracking.cc:953-1000, threshold mThEntropyReduction) -----------------------------------
 * For semantic key j with keypoint k, depth z = depth[j], classification entropy H and s2 = sigma2[k.octave] (the left
 * extractor's GetScaleSigmaSquares):
 *   valid iff z > 0 (NaN is invalid) and 0 <= octave < nlevels; an invalid key gets world = NaN x 3, reduction = NaN.
 *   world = Frame::UnprojectStereo (Frame.cc:631-645) in float: x = ((u - cx) * z) * invfx, y = ((v - cy) * z) * invfy,
 *           w_r = ((Rwc[r][0] * x + Rwc[r][1] * y) + Rwc[r][2] * z) + Ow[r], every operation rounded to float (cv::gemm).
 *   J     = computeStereoJacobianPose(fx, fy, mb, wX, wY, wZ) (sivo_helpers.cpp:64-88) in double, all zeros when wZ == 0.  As in
 *           the reference, it is given the WORLD point where the helper expects camera coordinates (equal at the identity pose).
 *   M     = [[S, S J^T], [J S, (J S) J^T + s2 I]] (9 x 9; S = sigma_cw), products summed over k in ascending order.
 *   MI    = 0.5 * log2((det S * det M33) / det M): det of the 3 x 3 by cofactors along the first row, of the 6 x 6 / 9 x 9 by LU
 *           with partial pivoting (the first row with the largest |a|; a zero pivot column is skipped).
 *   reduction = MI - H; key j is selected iff reduction > threshold (a NaN is never selected).
 * Steps 2-5 use no fused multiply-add, so every intermediate is the IEEE float / double result of the operation as written;
 * log2 is within an ulp of glibc's.  selected[0 .. n_selected) = the selected j, ascending: the order in which the reference
 * creates map points.  CreateNewKeyFrame's test for an existing map point stays with the caller (filter the selected list).
 * Any output may be NULL; the camera is copied at call time.  SIVO_EINVAL for a NULL handle, input or camera, or n < 0. */
typedef struct sivo_info_camera {          /* the Frame's own members */
  float fx, fy, cx, cy, invfx, invfy, mb;  /* Frame.cc:166-172 */
  float Rwc[9];                            /* mRwc, row-major */
  float Ow[3];                             /* mOw */
  double sigma_cw[36];                     /* mSigmacw, row-major 6x6 */
} sivo_info_camera;

/* Host buffers gathered per semantic key: kps = mvKeysSemantic, depth = mvDepth, entropy = mEntropy at ((int) y, (int) x); world
 * 3n floats, reduction n doubles, selected n ints.  Returns when done. */
int sivo_info_select(const sivo_orb_t* left, const sivo_keypoint* kps, const float* depth, const double* entropy, int n,
                     const sivo_info_camera* cam, double threshold, float* world, double* reduction, int* selected, int* n_selected);
/* The same selection on device buffers, e.g. the Frame tail's: semantic key j < *n_keep_device is extractor key keep_idx_device[j]
 * (j when keep_idx_device is NULL) of kps_device; its entropy is kp_entropy_device[keep_idx[j]] as sivo_segnet_semantic_keys_device
 * writes it, its depth depth_device[j] as sivo_stereo_match_device writes it.  Outputs as in the host form, each with room for
 * sivo_orb_capacity(left) keys; the values equal the host form's on the same keys gathered on the host, bit for bit.
 * *n_keep_device (int64) is read on the device and clamped to the capacity; a negative count (the -1 of
 * sivo_segnet_semantic_keys_device) writes nothing except *n_selected_device = -1.  A key index outside the capacity is invalid.
 * Ordering: runs on `stream` (NULL = the left extractor's stream) with no host synchronisation and no waits of its own, so every
 * input must be ordered before it on `stream` (on the Frame tail's stream they are), and the next sivo_orb_enqueue_device into
 * kps_device after it (sivo_orb_wait_for_stream(left, stream)). */
int sivo_info_select_device(const sivo_orb_t* left, const sivo_keypoint* kps_device, const double* kp_entropy_device,
                            const int* keep_idx_device, const long long* n_keep_device, const float* depth_device,
                            const sivo_info_camera* cam, double threshold, float* world_device, double* reduction_device,
                            int* selected_device, long long* n_selected_device, void* stream);
/* Test hook: the host form's world points and the three determinants per key (det S, det M33, det M; NaN for an invalid key). */
int sivo_dbg_info_terms(const sivo_orb_t* left, const sivo_keypoint* kps, const float* depth, int n, const sivo_info_camera* cam,
                        float* world, double* det_state, double* det_meas, double* det_joint);

/* ---- map points matched to a frame's semantic keys by projection: ORBmatcher::SearchByProjection(F, vpMapPoints, th) after
 * Frame::isInFrustum (Tracking::SearchLocalPoints, Tracking.cc:1033-1085) and SearchByProjection(CurrentFrame, LastFrame, th)
 * (Tracking::TrackWithMotionModel, Tracking.cc:704-746), with the Frame's grid (Frame.cc:205-223, 326-404) ------------------
 * Every operation is the IEEE float / double operation as written (no contracted multiply-add).  The rules, which
 * oracle/track_oracle.py restates:
 *   grid      key j goes to cell (round((x - min_x) * wInv), round((y - min_y) * hInv)), round = half away from zero, wInv =
 *             64.f / (max_x - min_x), hInv = 48.f / (max_y - min_y) in float; dropped outside 64 x 48; ascending j per cell.
 *   area      GetFeaturesInArea(x, y, r, minLevel, maxLevel): cells floor(((x - min_x) - r) * wInv) .. ceil(((x - min_x) + r) *
 *             wInv) with Frame.cc:334-358's early returns and clamps (same in y); walk ix ascending, then iy, then the cell's
 *             keys; levels filtered only when minLevel > 0 || maxLevel >= 0; kept iff |kp.x - x| < r && |kp.y - y| < r.
 *   Pc        ((R[r][0] X + R[r][1] Y) + R[r][2] Z) + t[r] in float (cv::gemm's 3 x 3 float form).
 *   frustum   (local-map search, isInFrustum(pMP, 0.5) + PredictScale) out if Pc_z < 0; invz = 1.0f / Pc_z; u = (fx Pc_x) invz + cx,
 *             v likewise; out unless min_x <= u <= max_x and min_y <= v <= max_y; dist = (float) sqrt of ((0 + a0 a0) + a1 a1) + a2 a2
 *             in double over a = pos - Ow in float (cv::norm); out unless 0.8f min_distance <= dist <= 1.2f max_distance; viewCos =
 *             (float)(((0 + a0 n0) + a1 n1) + a2 n2 in double / dist) (Mat::dot's scalar path for three floats, not pinnable
 *             against Python: only a viewCos within an ulp of 0.5 or 0.998 can depend on it); out if viewCos < 0.5f; level =
 *             ceil(logf(max_distance / dist) / logf(scale_factor)) clamped to [0, nlevels).  MapPoint.cc sees `using namespace
 *             std` through MapPoint.h -> KeyFrame.h -> ORBVocabulary.h -> DBoW2's TemplatedVocabulary.h, so PredictScale's log is
 *             the float overload; logf here is the correctly rounded float logarithm, within an ulp of glibc's.  projXR = u -
 *             mbf invz.
 *   local     per point in order, if in view: r = viewCos > 0.998 ? 2.5f : 4.0f, times th when th != 1; radius = r scale[level];
 *             candidates = area(u, v, radius, level - 1, level) minus keys held by an observed point and keys with u_right > 0
 *             and |projXR - u_right| > radius; best / second fold as ORBmatcher.cc:86-113; accepted iff bestDist <= 100 and not
 *             (bestLevel == bestLevel2 && bestDist > nnratio bestDist2); an accepted point takes its key (F.mvpMapPoints[bestIdx] =
 *             pMP), which blocks the key for every later point iff the point is observed.
 *   last      twc = -Rcw^T tcw (each entry the double sum of the three products, rounded to float: cv::gemm with GEMM_1_T); tlc =
 *             Rlw twc + tlw in the Pc form; forward iff tlc_z > mb, backward iff -tlc_z > mb.  Per point in order: invzc = (float)
 *             (1.0 / Pc_z) in double, out if invzc < 0; u, v with invzc, out of bounds as above; o = octave; radius = th scale[o];
 *             area(u, v, radius, o, -1) forward, (0, o) backward, else (o - 1, o + 1); the stereo gate uses ur = u - mbf invzc;
 *             best distance only, accepted iff <= 100; the key is taken as above (a key taken by an unobserved point can be taken
 *             again: the last writer wins).  Rotation check: rot = angle - key angle, + 360 if negative; bin = roundf(rot * (1.f /
 *             30)), 30 -> 0 (so only bins 0..12 are used, as in the reference); ComputeThreeMaxima with its 0.1f * max1 rule; every
 *             entry of every other bin frees its key and decrements the count, duplicates included.
 *   NaN       a point whose u, v, viewCos or level quotient is NaN is not in view (the reference converts a NaN to int there).
 *   angles    key angles (kp.angle, both searches) and last-frame point angles must be finite and in [0, 360] (-0.0 included),
 *             which keeps rot in [0, 360] and every bin in 0..12 (the reference asserts 0 <= bin < 30, ORBmatcher.cc:1390).  The
 *             host forms return SIVO_ERANGE for any other angle.  The device forms put a key with such an angle in no cell (as
 *             a key index outside the capacity) and do not search a last-frame point with one.  Extractor keys satisfy the rule.
 * Map-point order and claims make the result sequential; the device walks the points in order in one block and re-searches only
 * the points whose best (or, local, second-best) key an earlier point took.  tests/test_gpu_track_edges.py holds the device
 * forms to oracle/track_oracle.py on constructed worst cases: crowded windows, exact ties, every decision boundary, long claim
 * chains, the limits and a seeded differential fuzz. */
typedef struct sivo_track_frame {          /* the current Frame's members */
  float fx, fy, cx, cy, mb, mbf;
  float min_x, max_x, min_y, max_y;        /* mnMinX, mnMaxX, mnMinY, mnMaxY (ComputeImageBounds) */
  float Rcw[9], tcw[3], Ow[3];             /* mRcw row-major, mtcw, mOw */
} sivo_track_frame;

typedef struct sivo_map_point {            /* 80 bytes, one per map point */
  uint8_t desc[32];                        /* GetDescriptor */
  float pos[3], normal[3];                 /* GetWorldPos, GetNormal */
  float min_distance, max_distance;        /* mfMinDistance, mfMaxDistance: the search applies 0.8f / 1.2f itself */
  int32_t observed;                        /* Observations() > 0 */
  int32_t octave;                          /* last-frame search: LastFrame.mvKeysSemantic[i].octave */
  float angle;                             /* last-frame search: LastFrame.mvKeysSemantic[i].angle */
  int32_t reserved;
} sivo_map_point;

/* SearchLocalPoints' isInFrustum loop and SearchByProjection(F, vpMapPoints, th) on device buffers.  Semantic key j <
 * *n_keep_device is extractor key keep_idx_device[j] (j when NULL) of kps_device / desc_device (the Frame tail's buffers);
 * u_right_device[j] is its mvRight.  blocked_device[j] (u8, may be NULL) = mvpMapPoints[j] && Observations() > 0 on entry.  The
 * points are mvpLocalMapPoints in order, without the ones SearchLocalPoints skips (already seen by the frame, bad).  Outputs (any
 * may be NULL): in_view_device[i] (u8, n_points) = isInFrustum's result (the caller's IncreaseVisible); match_device[j] (int,
 * sivo_orb_capacity(left)) = the point this call gave key j, or -1; *n_matches_device (int64) = SearchByProjection's return.
 * *n_keep_device is clamped to the capacity; a negative count writes only *n_matches_device = -1.  A key index outside the
 * capacity is in no cell.  Runs on `stream` (NULL = the left extractor's stream) with no waits of its own and no host
 * synchronisation.  SIVO_EINVAL for NULL handles or inputs, n_points < 0, th <= 0, nnratio not finite, or max <= min in
 * the bounds. */
int sivo_search_local_points_device(const sivo_orb_t* left, const sivo_keypoint* kps_device, const uint8_t* desc_device,
                                    const int* keep_idx_device, const long long* n_keep_device, const float* u_right_device,
                                    const uint8_t* blocked_device, const sivo_map_point* points_device, int n_points,
                                    const sivo_track_frame* frame, float th, float nnratio, uint8_t* in_view_device, int* match_device,
                                    long long* n_matches_device, void* stream);
/* SearchByProjection(CurrentFrame, LastFrame, th) (stereo) on device buffers, keys as above.  The points are the last frame's
 * non-NULL, non-outlier map points in key order, each with its key's octave and angle; no key is blocked on entry (Tracking
 * clears mvpMapPoints before both calls).  Rlw / tlw: the last frame's pose (host, row-major 3 x 3 and 3).  match_device /
 * n_matches_device as above.  A point whose octave is outside [0, nlevels), or whose angle breaks the angle rule, is never
 * matched (the host form refuses it). */
int sivo_search_last_frame_device(const sivo_orb_t* left, const sivo_keypoint* kps_device, const uint8_t* desc_device,
                                  const int* keep_idx_device, const long long* n_keep_device, const float* u_right_device,
                                  const sivo_map_point* points_device, int n_points, const sivo_track_frame* frame, const float* Rlw,
                                  const float* tlw, float th, int* match_device, long long* n_matches_device, void* stream);
/* Host forms: n keys gathered per semantic key (mvKeysSemantic, mDescriptorsSemantic n x 32, mvRight, blocked may be NULL), points
 * on the host; outputs in_view (n_points), match (n), *n_matches, any may be NULL.  They stage the inputs and run the device
 * forms' kernels, then synchronise.  SIVO_EINVAL as above and for n < 0; SIVO_ERANGE for a last-frame octave outside [0, nlevels)
 * and for an angle that breaks the angle rule.  At most 40,960 keys (the ordered pass keeps 5 bytes per key in shared memory). */
int sivo_search_local_points(const sivo_orb_t* left, const sivo_keypoint* kps, const uint8_t* desc, const float* u_right,
                             const uint8_t* blocked, int n, const sivo_map_point* points, int n_points, const sivo_track_frame* frame,
                             float th, float nnratio, uint8_t* in_view, int* match, int* n_matches);
int sivo_search_last_frame(const sivo_orb_t* left, const sivo_keypoint* kps, const uint8_t* desc, const float* u_right, int n,
                           const sivo_map_point* points, int n_points, const sivo_track_frame* frame, const float* Rlw,
                           const float* tlw, float th, int* match, int* n_matches);
/* Test hook: GetFeaturesInArea on the device grid of n host keys within the bounds.  Query q is (xyr[3 q], xyr[3 q + 1],
 * xyr[3 q + 2], levels[2 q], levels[2 q + 1]); its list is idx[offsets[q] .. offsets[q + 1]).  SIVO_ERANGE (offsets written) if
 * idx_cap is too small. */
int sivo_dbg_features_in_area(const sivo_orb_t* left, const sivo_keypoint* kps, int n, float min_x, float max_x, float min_y,
                              float max_y, const float* xyr, const int* levels, int n_query, int* offsets, int* idx, int idx_cap);

/* ---- the frame pose: Optimizer::PoseOptimization (Optimizer.cc:273-491) with g2o's Levenberg-Marquardt, and the pose's
 * marginal covariance (computeMarginals, :480-487), as Tracking runs it after each projection search ----------------------------
 * Every operation is the IEEE float / double operation as written (no contracted multiply-add).  oracle/pose_oracle.py restates
 * the rules and the reference facts kept (its header lists them with their g2o sources); in short:
 *   edges     one per semantic key j with a map point (xw[3 j] not NaN), in key order; stereo iff u_right[j] >= 0 is not false
 *             (mvRight < 0: mono).  Omega = I * mvInvLevelSigma2[octave] (the left extractor's table), Huber deltas sqrt(5.991f)
 *             and sqrt(7.815f) in float.  Mono u = (x / z) fx + cx in double; stereo invz = (float)(1.0 / z), u = ((x invz) fx) +
 *             cx, ur = u - mbf invz.  Jacobians as g2o's linearizeOplus, update [omega, upsilon]; robust weighting rho1 Omega only.
 *   LM        tau 1e-5, lambda re-initialised per optimize(); <= 10 trials after a failure; scale = x . (lambda x + b) + 1e-3;
 *             Terminate on qmax == 10, rho == 0 or a non-finite lambda; a failed factorisation sets tempChi = DBL_MAX and keeps
 *             the last solved x (zeros before the first).  oplus = SE3Quat::exp(delta) * T with its theta < 1e-5 branch.
 *   rounds    4 rounds of 10 iterations, each from the INPUT pose; only stereo edges are classified (outlier iff (float) chi2 >
 *             7.815f), an inlier with the chi2 the last error pass left (possibly a rejected trial's), an outlier recomputed at
 *             the round's estimate; stereo kernels removed after round 2; stop after a round when there are < 10 edges.  Below
 *             3 edges: n_good = 0, the pose untouched.
 *   result    Tcw = the quaternion's toRotationMatrix and t rounded to float; Ow = -Rcw^T tcw as Frame::UpdatePoseMatrices;
 *             sigma_cw = the inverse of the last linearisation's H (LL^T in natural order, then MarginalCovarianceCholesky's
 *             recursion), sigma_valid = 0 (sigma_cw zeros: keep the prior) when a pivot is not > 0 or the last round had no
 *             inlier edge.  n_good = n_initial - n_bad of the last round run.
 *   NaN rule  an edge is valid at a pose iff its chi2 and 1 / z^2 are finite; an invalid edge adds nothing to H, b or chi2 and
 *             is an outlier when classified.
 *   order     sums over edges run in a fixed tree: thread t of 256 sums edges t, t + 256, ...; xor shuffles 16 .. 1 in each warp;
 *             the 8 warp totals folded by halves.  The reference sums in key order; the two agree to rounding.
 * Not pinned to the reference (not buildable here): CHOLMOD's ordering, Eigen's operation orders, sin / cos / pow. */
typedef struct sivo_pose_result {
  float Tcw[12];                           /* 3 x 4 row-major [Rcw | tcw]: the next call's Tcw_in */
  double q[4], t[3];                       /* the SE3Quat: quaternion (x, y, z, w) and translation */
  float Rcw[9], tcw[3], Rwc[9], Ow[3];     /* sivo_track_frame's Rcw / tcw / Ow, sivo_info_camera's Rwc / Ow */
  double sigma_cw[36];                     /* mSigmacw, row-major 6 x 6 [omega, upsilon] (sivo_info_camera.sigma_cw) */
  int32_t sigma_valid, n_initial, n_bad, n_good, rounds_run, reserved;  /* n_good: PoseOptimization's return */
} sivo_pose_result;

/* PoseOptimization on device buffers.  Semantic key j < *n_keep_device is extractor key keep_idx_device[j] (j when NULL) of
 * kps_device; u_right_device[j] is its mvRight, xw_device[3 j ..] its map point's world position (NaN x: no map point, e.g.
 * filled by sivo_pose_gather_device).  Tcw_in_device: 12 floats, the frame's 3 x 4 pose (a sivo_pose_result's Tcw may be
 * passed, that of result_device itself included: the pose is read before the result is written).  Writes *result_device and
 * outlier_device[j] for j < the count (u8, sivo_orb_capacity(left) room; may be NULL): 0 for a key without a map point, where
 * the reference leaves mvbOutlier as the caller had it, so the buffer is the call's whole output.  A key index outside the capacity, or a key with an octave outside the extractor's levels, has no edge.  The count is
 * clamped to the capacity; a negative count (the -1 of sivo_segnet_semantic_keys_device) writes only result_device->n_good =
 * -1.  One block runs the whole optimisation.  Runs on `stream` (NULL = the left extractor's stream) with no waits of its own
 * and no host synchronisation.  SIVO_EINVAL for NULL handles or inputs, or fx, fy, mbf not finite and positive, cx, cy not finite. */
int sivo_pose_optimize_device(const sivo_orb_t* left, const sivo_keypoint* kps_device, const int* keep_idx_device,
                              const long long* n_keep_device, const float* u_right_device, const float* xw_device, float fx, float fy,
                              float cx, float cy, float mbf, const float* Tcw_in_device, sivo_pose_result* result_device,
                              uint8_t* outlier_device, void* stream);
/* For semantic keys j < *n_keep_device: if 0 <= match_device[j] < n_points, xw_device[3 j ..] = points_device[match[j]].pos; other
 * entries are left alone, so matches of several searches merge into one array (as mvpMapPoints).  Same stream and ordering
 * rules; SIVO_EINVAL for NULL handles or buffers or n_points < 0. */
int sivo_pose_gather_device(const sivo_orb_t* left, const int* match_device, const long long* n_keep_device,
                            const sivo_map_point* points_device, int n_points, float* xw_device, void* stream);
/* Host form: n keys gathered per semantic key (mvKeysSemantic, mvRight, xw), the pose as 12 host floats; result and outlier (n)
 * on the host.  It stages the inputs, runs the device form's kernel and synchronises.  SIVO_EINVAL as above and for n < 0;
 * SIVO_ERANGE for a key with a point whose octave is outside the extractor's levels. */
int sivo_pose_optimize(const sivo_orb_t* left, const sivo_keypoint* kps, const float* u_right, const float* xw, int n, float fx,
                       float fy, float cx, float cy, float mbf, const float* Tcw_in, sivo_pose_result* result, uint8_t* outlier);
/* Test hook: one linearisation pass of the kernel at pose7 = (qx, qy, qz, qw, tx, ty, tz) over the host keys' edges, with the
 * stereo kernels on iff robust_stereo, edges j with level1[j] != 0 left out of the sums (level1 may be NULL).  Per key (NaN for a
 * key without an edge): err[3 j ..], chi2[j], rho[2 j ..] = (rho0, rho1), jac[18 j ..] (3 x 6 row-major; a mono edge's third row
 * zero).  H (36, row-major), b (6) and *chi (the robust chi2) as the kernel's reduction produces them.  Any output may be NULL. */
int sivo_dbg_pose_system(const sivo_orb_t* left, const sivo_keypoint* kps, const float* u_right, const float* xw, int n, float fx,
                         float fy, float cx, float cy, float mbf, const double* pose7, int robust_stereo, const uint8_t* level1,
                         double* err, double* chi2, double* rho, double* jac, double* H, double* b, double* chi);

/* Test hook: sivo_pose_optimize run by the traced instantiation of its kernel, which also records the optimisation as thread 0
 * runs it.  Per trial (after its lambda update): kind SIVO_POSE_TRACE_TRIAL, round, iteration, trial (qmax before the increment),
 * ok2 (the factorisation succeeded), accepted, current (currentChi before the update), temp (DBL_MAX after a failed
 * factorisation), lam / ni before and after, rho, x (the solver's buffer used) and the trial pose q, t.  Before it, one record
 * per transcendental call, in call order, with its argument and result: the theta >= 1e-5 branch of oplus calls sin(theta),
 * cos(theta) and pow(theta, 3) (arg = theta); an accepted trial calls pow(2 rho - 1, 3) (arg = 2 rho - 1).  Per round run, after
 * its classification: SIVO_POSE_TRACE_ROUND with n_active (the round's level-0 edges), n_bad and robust_stereo (the round's
 * stereo kernels).  At most SIVO_POSE_TRACE_MAX records (4 rounds x 10 iterations x 10 trials of at most 5, plus 4).  Writes
 * the first trace_cap records to trace (may be NULL when trace_cap is 0) and returns the number recorded, or a negative error
 * code as sivo_pose_optimize; outlier may be NULL. */
#define SIVO_POSE_TRACE_TRIAL 0
#define SIVO_POSE_TRACE_ROUND 1
#define SIVO_POSE_TRACE_SIN 2
#define SIVO_POSE_TRACE_COS 3
#define SIVO_POSE_TRACE_POW_THETA 4
#define SIVO_POSE_TRACE_POW_RHO 5
#define SIVO_POSE_TRACE_MAX (4 + 4 * 10 * 10 * 5)
typedef struct sivo_pose_trace_rec {
  int32_t kind, round, iteration, trial;
  int32_t ok2, accepted, n_active, n_bad, robust_stereo, reserved;
  double current, temp, lam_before, ni_before, lam_after, ni_after, rho;
  double x[6], q[4], t[3];
  double arg, value;
} sivo_pose_trace_rec;
int sivo_dbg_pose_trace(const sivo_orb_t* left, const sivo_keypoint* kps, const float* u_right, const float* xw, int n, float fx,
                        float fy, float cx, float cy, float mbf, const float* Tcw_in, sivo_pose_result* result, uint8_t* outlier,
                        sivo_pose_trace_rec* trace, int trace_cap);
/* Test hook: the kernel's own SE3Quat functions on n >= 1 host entries, one thread each on `device`.  Entry i: se3[7 i ..] =
 * to_se3quat(T[12 i ..]) as (qx, qy, qz, qw, tx, ty, tz); up[7 i ..] = oplus(d[6 i ..], that pose) as a trial step computes it;
 * tv[4 i ..] = (theta, sin theta, cos theta, pow(theta, 3)) of that oplus (the last three NaN on the theta < 1e-5 branch);
 * res[i] = the result's pose fields as the kernel writes them from that estimate (sigma and counts unwritten). */
int sivo_dbg_pose_se3(int device, int n, const float* T, const double* d, double* se3, double* up, double* tv, sivo_pose_result* res);

/* ---- a keyframe's new map points: LocalMapping::CreateNewMapPoints (LocalMapping.cc:198-472) with ORBmatcher::
 * SearchForTriangulation (ORBmatcher.cc:631-785, ORBmatcher(0.6, false): no orientation check), CheckDistEpipolarLine
 * (:137-159), ComputeF12 (LocalMapping.cc:639-654) and SIVO's CheckSemantics (:474-545), stereo only -------------------------
 * Every operation is the IEEE float / double operation as written (no contracted multiply-add).  oracle/mapping_oracle.py restates
 * the rule and lists every reference fact kept; in short:
 *   walk      current-keyframe key j (no map point on entry) visits the neighbours in order and stops at its first created point.
 *             A neighbour with (float) norm(Ow2 - Ow1) < mb is skipped.  Key results do not depend on one another: the reference
 *             never sets vbMatched2, so one neighbour key may be matched (and get points) from several current keys.
 *   match     candidates: the neighbour's keys with node == node[j] >= 0 and no map point on entry (node -1: not in mFeatVec);
 *             Hamming distance <= TH_LOW (50); if both keys are mono, (ex - x2)^2 + (ey - y2)^2 < 100 scale[octave2] rejects (the
 *             scale factor, not squared); CheckDistEpipolarLine in float with den == 0 rejecting and dsqr < 3.84 sigma2 in double.
 *             The best is the smallest distance, the LATER candidate on ties (the reference's `dist > bestDist` skip).
 *   checks    in the reference's order: parallax (cos(2 atan2(mb / 2, depth)) as the float overloads, the second keyframe's only in
 *             the `else if`), w == 0, z1 <= 0, z2 <= 0, the reprojection errors (5.991 / 7.8 sigma2 in double; the neighbour's
 *             stereo error with the current keyframe's mbf), scale consistency (1.5f scale_factor).
 *   SVD       the triangulation's right singular vector is a documented rule, not cv::SVD's float Jacobi: one-sided Jacobi in
 *             double on A's columns (pairs (0,1) (0,2) (0,3) (1,2) (1,3) (2,3), a pair rotated only while |gamma| > 2^-52
 *             sqrt(alpha beta), at most 30 sweeps, stop after a sweep without a rotation), the column of least norm (first on
 *             ties); rounded to float, w == 0 rejects, x = v[0..2] / v[3] in float.
 *   semantic  current key: depth > 0, class <= max_static_class, (double) confidence >= (float) th_confidence, and not
 *             MI - H < (float) th_entropy_reduction, with MI of the triangulated WORLD point, sigma2[octave] and sigma_cw (a NaN
 *             reduction passes).  Neighbour key: its class.  Created iff the two classes are equal and not 255 (VOID).
 * A key whose octave is outside the extractor's levels never takes part (the reference would index out of its tables). */
typedef struct sivo_keyframe_keys {        /* one keyframe's semantic keys, sivo_orb_capacity(left) entries per array */
  const sivo_keypoint* kps;                /* mvKeysSemantic */
  const uint8_t* desc;                     /* mDescriptorsSemantic, 32 bytes per key */
  const float* u_right;                    /* mvRight (< 0: mono) */
  const float* depth;                      /* mvDepth */
  const uint8_t* kp_class;                 /* mClasses, mConfidence, mEntropy at ((int) y, (int) x) */
  const double* kp_conf;
  const double* kp_entropy;
  const int32_t* node;                     /* the key's mFeatVec node (DBoW2, levelsup 4); -1 for none */
  const uint8_t* has_point;                /* GetMapPoint(i) != NULL on entry */
  const long long* count;                  /* int64 number of keys */
  float Rcw[9], tcw[3], Ow[3];             /* GetRotation (row-major), GetTranslation, GetCameraCenter (host values) */
} sivo_keyframe_keys;

typedef struct sivo_mapping_params {       /* the keyframes' shared camera and SIVO's thresholds */
  float fx, fy, cx, cy, invfx, invfy, mb, mbf;
  double sigma_cw[36];                     /* the current keyframe's mSigmacw, row-major 6 x 6 */
  int32_t max_static_class;                /* Classes::TERRAIN = 8 in the reference */
  float th_confidence, th_entropy_reduction;  /* mThConfidence, mThEntropyReduction */
  int32_t reserved;
} sivo_mapping_params;

/* KeyFrame's copy of the Frame's semantic keys: for j < *n_keep_device (clamped to the capacity), with k = keep_idx_device[j] (j
 * when NULL), out_kps[j] = kps[k], out_desc[32 j ..] = desc[32 k ..], out_u_right[j] = u_right[j], out_depth[j] = depth[j],
 * out_class / out_conf / out_entropy[j] = kp_class / kp_conf / kp_entropy[k]; *out_count = the clamped count (-1 for a negative
 * count, which writes nothing else).  A key index outside the capacity gives octave -1 (the key never takes part).  Outputs hold
 * sivo_orb_capacity(left) keys and belong to the caller, so the next sivo_orb_enqueue_device does not overwrite them.  Runs on
 * `stream` (NULL = the left extractor's stream) with no waits and no host synchronisation; the inputs must be ordered before it
 * on that stream, as for the other Frame-tail calls.  SIVO_EINVAL for NULL handles, inputs or outputs. */
int sivo_keyframe_gather_device(const sivo_orb_t* left, const sivo_keypoint* kps_device, const uint8_t* desc_device,
                                const int* keep_idx_device, const long long* n_keep_device, const float* u_right_device,
                                const float* depth_device, const uint8_t* kp_class_device, const double* kp_conf_device,
                                const double* kp_entropy_device, sivo_keypoint* out_kps, uint8_t* out_desc, float* out_u_right,
                                float* out_depth, uint8_t* out_class, double* out_conf, double* out_entropy, long long* out_count,
                                void* stream);
/* CreateNewMapPoints of keyframe kf1 against neighbours[0 .. n_neighbours) (GetBestCovisibilityKeyFrames order, at most 32) on
 * device buffers.  Outputs, each may be NULL, for current keys j < kf1's count (sivo_orb_capacity(left) room):
 * created_nb_device[j] = the neighbour whose pair created j's point, or -1; created_idx_device[j] = that neighbour's key;
 * world_device[3 j ..] = the point (NaN when none); created_list_device[2 e ..] = (neighbour, key j) of the e-th point created, in
 * the reference's order (neighbour-major, j ascending: mlpRecentAddedMapPoints); *n_created_device (int64) its length.  Counts are
 * clamped to the capacity; a negative count (the -1 of sivo_segnet_semantic_keys_device) in any keyframe writes only
 * *n_created_device = -1.  Runs on `stream` (NULL = the left extractor's stream) with no waits and no host synchronisation.  It
 * reads only the extractor's scale tables: LocalMapping's thread may run it concurrently with Tracking's calls on the same extractor.  SIVO_EINVAL for NULL
 * handles or inputs, n_neighbours outside [0, 32]. */
int sivo_create_map_points_device(const sivo_orb_t* left, const sivo_keyframe_keys* kf1, const sivo_keyframe_keys* neighbours,
                                  int n_neighbours, const sivo_mapping_params* params, int* created_nb_device,
                                  int* created_idx_device, float* world_device, int* created_list_device, long long* n_created_device,
                                  void* stream);
/* Host form: every sivo_keyframe_keys pointer (count included) is a host array of its own count's keys; outputs per current key
 * (n1 = kf1's count) and created_list 2 n1 ints, *n_created.  It stages the inputs, runs the device form's kernels and
 * synchronises. */
int sivo_create_map_points(const sivo_orb_t* left, const sivo_keyframe_keys* kf1, const sivo_keyframe_keys* neighbours, int n_neighbours,
                           const sivo_mapping_params* params, int* created_nb, int* created_idx, float* world, int* created_list,
                           long long* n_created);
/* Test hook: the host form, every key searched (the production path skips a key whose depth, class or confidence already
 * rules it out), plus per (neighbour i, key j) at [i n1 + j]: match = SearchForTriangulation's vMatchedPairs partner or -1;
 * stage = where the reference's loop ends for the pair (SIVO_MAP_STAGE_*); reduction = MI - H (NaN unless computed). */
enum {
  SIVO_MAP_STAGE_HAS_POINT = 0, SIVO_MAP_STAGE_BASELINE, SIVO_MAP_STAGE_NO_MATCH, SIVO_MAP_STAGE_PARALLAX, SIVO_MAP_STAGE_W_ZERO,
  SIVO_MAP_STAGE_Z1, SIVO_MAP_STAGE_Z2, SIVO_MAP_STAGE_REPROJ1, SIVO_MAP_STAGE_REPROJ2, SIVO_MAP_STAGE_SCALE,
  SIVO_MAP_STAGE_SEMANTIC, SIVO_MAP_STAGE_CREATED
};
int sivo_dbg_create_map_points(const sivo_orb_t* left, const sivo_keyframe_keys* kf1, const sivo_keyframe_keys* neighbours,
                               int n_neighbours, const sivo_mapping_params* params, int* match, int* stage, double* reduction,
                               int* created_nb, int* created_idx, float* world, int* created_list, long long* n_created);

/* ---- a keyframe's map points fused with its neighbours': ORBmatcher::Fuse(pKF, vpMapPoints, th) (ORBmatcher.cc:787-930) as
 * LocalMapping::SearchInNeighbors (LocalMapping.cc:547-637) runs it, over every target keyframe at once ------------------------
 * Every operation is the IEEE float / double operation as written (no contracted multiply-add).  oracle/fuse_oracle.py restates
 * the rule and lists the reference facts kept; per (target k, point i):
 *   Pc        the projection searches' gemm form with target k's pose; out (DEPTH) if Pc_z < 0.0f (z = +-0 carries on).
 *   image     invz = 1 / Pc_z, x = Pc_x invz, u = fx x + cx (v likewise), all float; out (IMAGE) unless KeyFrame::IsInImage:
 *             min_x <= u < max_x && min_y <= v < max_y (strict upper bounds, unlike Frame::isInFrustum; a NaN is out).
 *             ur = u - mbf invz.
 *   distance  PO = pos - Ow in float, dist3D as the projection searches' cv::norm; out (DISTANCE) if dist3D < 0.8f min_distance
 *             || dist3D > 1.2f max_distance.
 *   angle     out (ANGLE) if PO . normal (Mat::dot, double, as the projection searches) < 0.5 * dist3D in double.  A NaN dot
 *             passes, as in the reference.
 *   level     PredictScale(dist3D) with the projection searches' rule; a NaN quotient searches nothing (NO_CANDIDATE).  radius =
 *             th scale[level] in float.
 *   window    KeyFrame::GetFeaturesInArea(u, v, radius): the projection searches' grid and walk, no level filter.  An empty
 *             window ends at NO_CANDIDATE.
 *   keys      a key in the window is a candidate iff level - 1 <= octave <= level, 0 <= octave < nlevels (the reference would
 *             read mvInvLevelSigma2[-1] for sivo_keyframe_gather_device's octave -1 at level 0), and e2 invSigma2[octave] in
 *             float, compared in double, is not above 7.8 for a stereo key (u_right >= 0; e2 = (ex^2 + ey^2) + er^2) or 5.99 for
 *             a mono one (a NaN u_right is mono; e2 = ex^2 + ey^2), with ex = u - x, ey = v - y, er = ur - u_right.
 *   best      the first strictly smaller Hamming distance in walk order, from 256; MATCHED iff it is <= TH_LOW (50), else
 *             ABOVE_TH_LOW.
 *   angles    key angles follow the projection searches' angle rule: a key with another angle is in no cell (the host form
 *             returns SIVO_ERANGE).  Extractor keys satisfy it.
 * Fuse claims no key: a pair's decision reads only the point's position, normal, distances and descriptor and the target's keys
 * and pose, so one warp decides each pair independently.  Replay contract: during SearchInNeighbors only a point's descriptor
 * can change (MapPoint::Replace ends with ComputeDistinctiveDescriptors on the survivor; UpdateNormalAndDepth runs after both
 * phases).  A caller that walks the pairs in the reference's order (phase 1: target-major, the current keyframe's points in
 * key order; phase 2: the current keyframe against the deduplicated candidates) and
 *   1. skips a point that is bad now or already in target k now,
 *   2. applies match[k n_points + i] to any other point (the reference's Replace / AddObservation / AddMapPoint), and
 *   3. searches again any point whose descriptor now differs from the one it was searched with (only the survivor of a Replace
 *      in an earlier target, so never in phase 2), applying that result instead,
 * reproduces the sequential loop exactly. */
typedef struct sivo_fuse_camera {          /* the keyframes' shared members */
  float fx, fy, cx, cy, mbf;
  float min_x, max_x, min_y, max_y;        /* mnMinX, mnMaxX, mnMinY, mnMaxY */
} sivo_fuse_camera;
/* Fuse of points_device[0 .. n_points) into targets[0 .. n_targets) on device buffers.  Target k: its kps / desc / u_right /
 * count (device, sivo_orb_capacity(left) keys, as sivo_keyframe_gather_device writes them) and its pose (Rcw, tcw, Ow); the
 * other pointers may be NULL.  A point reads only desc, pos, normal, min_distance and max_distance.  Outputs, row k at k n_points:
 * match_device[k n_points + i] = the key point i fuses with in target k, or -1; dist_device[...] (may be NULL) = the best
 * distance (256 when no key passed).  Counts are clamped to the capacity; a target with a negative count gets -1 (and 256) in
 * its whole row.  Targets go 64 to a launch.  Runs on `stream` (NULL = the left extractor's stream) with no waits of its own and
 * no host synchronisation.  SIVO_EINVAL for NULL handles or inputs, n_targets < 0, n_points < 0, n_targets n_points > INT_MAX,
 * th <= 0 or not finite, or max <= min in the bounds. */
int sivo_fuse_device(const sivo_orb_t* left, const sivo_keyframe_keys* targets, int n_targets, const sivo_fuse_camera* cam,
                     const sivo_map_point* points_device, int n_points, float th, int* match_device, int* dist_device, void* stream);
/* Host form: every target's kps / desc / u_right / count are host arrays of its own count's keys; points, match and dist (may be
 * NULL) on the host.  It stages the inputs, runs the device form's kernels and synchronises.  SIVO_EINVAL as above; SIVO_ERANGE
 * for a key angle that breaks the angle rule. */
int sivo_fuse(const sivo_orb_t* left, const sivo_keyframe_keys* targets, int n_targets, const sivo_fuse_camera* cam,
              const sivo_map_point* points, int n_points, float th, int* match, int* dist);
/* Test hook: the host form plus stage[k n_points + i] = where the reference's loop ends for the pair (SIVO_FUSE_STAGE_*; -1 for a
 * target with a negative count). */
enum {
  SIVO_FUSE_STAGE_DEPTH = 0, SIVO_FUSE_STAGE_IMAGE, SIVO_FUSE_STAGE_DISTANCE, SIVO_FUSE_STAGE_ANGLE, SIVO_FUSE_STAGE_NO_CANDIDATE,
  SIVO_FUSE_STAGE_ABOVE_TH_LOW, SIVO_FUSE_STAGE_MATCHED
};
int sivo_dbg_fuse(const sivo_orb_t* left, const sivo_keyframe_keys* targets, int n_targets, const sivo_fuse_camera* cam,
                  const sivo_map_point* points, int n_points, float th, int* match, int* dist, int* stage);

/* ---- the DBoW2 vocabulary: TemplatedVocabulary<FORB::TDescriptor, FORB>::loadFromTextFile (DBoW2 TemplatedVocabulary.h:1338-1420)
 * ---------------------------------------------------------------------------------------------------------------------------------
 * Text form: line 1 is `k L scoring weighting`; every further line is one node, id = its line number (the root is 0 and has no
 * line): `parent isLeaf d0 .. d31 weight`.  A descriptor byte is (unsigned char) of its integer token (FORB::fromString); the
 * weight is a double; tokens after the weight are ignored; leaves (isLeaf > 0) get word ids in id order; a node's children keep
 * id order, which decides ties in the descent.  Refused with SIVO_EFORMAT:
 *   header    where the reference returns false: k < 0 || k > 20 || L < 1 || L > 10 || scoring outside [0, 5] || weighting outside
 *             [0, 3]; also fewer than four integer tokens.
 *   node      a parent that is not an earlier node, a parent that is a leaf, fewer than 34 integer tokens before the weight or no
 *             weight (a truncated final line included), a non-leaf node without children (the reference would index its empty child
 *             list), an empty tree.
 *   blank     trailing whitespace-only lines add no node (the reference's eof loop would append a phantom child of the root with an
 *             indeterminate descriptor); a blank line followed by a further node is refused (the reference would shift every later
 *             id).
 * Enum values are DBoW2's: weighting TF_IDF 0, TF 1, IDF 2, BINARY 3; scoring L1_NORM 0, L2_NORM 1, CHI_SQUARE 2, KL 3,
 * BHATTACHARYYA 4, DOT_PRODUCT 5.  The device copy holds 32 descriptor bytes, a child offset, a child id and a word id per node and
 * a double per word (about 56 MB for ORBvoc).  A vocabulary is read-only once created: any number of threads may use it at once. */
typedef struct sivo_vocabulary sivo_vocabulary_t;
enum { SIVO_WEIGHTING_TF_IDF = 0, SIVO_WEIGHTING_TF = 1, SIVO_WEIGHTING_IDF = 2, SIVO_WEIGHTING_BINARY = 3 };
enum { SIVO_SCORING_L1_NORM = 0, SIVO_SCORING_L2_NORM = 1, SIVO_SCORING_CHI_SQUARE = 2, SIVO_SCORING_KL = 3,
       SIVO_SCORING_BHATTACHARYYA = 4, SIVO_SCORING_DOT_PRODUCT = 5 };
/* Loads a text vocabulary onto `device`.  SIVO_ENOENT if the file cannot be read, SIVO_EFORMAT as above. */
int sivo_vocabulary_load_text(const char* path, int device, sivo_vocabulary_t** out);
/* The same tree as arrays of n_nodes entries indexed by node id, the root at 0 (its entries are ignored): parent, is_leaf (nonzero:
 * leaf), desc (32 bytes per node), weight.  The text loader is a parser in front of this call; the same rules apply. */
int sivo_vocabulary_create(int device, int k, int L, int scoring, int weighting, const int32_t* parent, const uint8_t* is_leaf,
                           const uint8_t* desc, const double* weight, int n_nodes, sivo_vocabulary_t** out);
/* n_nodes counts the root; any output may be NULL. */
int sivo_vocabulary_info(const sivo_vocabulary_t* voc, int* k, int* L, int* scoring, int* weighting, int* n_nodes, int* n_words);
void sivo_vocabulary_destroy(sivo_vocabulary_t* voc);
/* Test hook: the text parser and the checks without a device.  header[4] = k, L, scoring, weighting; *n_nodes (root included);
 * the arrays as sivo_vocabulary_create takes them (the root's entries: parent -1, not a leaf, zero descriptor and weight), written
 * only when capacity >= *n_nodes (each may be NULL); SIVO_ERANGE with *n_nodes set when capacity is smaller. */
int sivo_dbg_vocabulary_parse(const char* path, int* header, int* n_nodes, int32_t* parent, uint8_t* is_leaf, uint8_t* desc,
                              double* weight, int capacity);

/* ---- Frame::ComputeBoW / KeyFrame::ComputeBoW: TemplatedVocabulary::transform(features, v, fv, levelsup) (TemplatedVocabulary.h:
 * 1127-1195) and the per-feature descent (:1218-1259) over a frame's semantic descriptors --------------------------------------
 * Every operation is the IEEE double operation as written (no contracted multiply-add).  oracle/bow_oracle.py restates the rules:
 *   descent   from the root, each level takes the child with the smallest Hamming distance, compared with a strict `<` in child
 *             order (the first child wins ties), until a node without children (a leaf).  The node recorded is the one reached at
 *             level nid_level = L - levelsup; the root (0) when nid_level <= 0; the leaf itself when the path ends above
 *             nid_level (the reference leaves nid uninitialised there: in practice the previous feature's node).
 *   keys      a key enters the BowVector and the FeatureVector only when its word's weight w > 0 (stopped words have w = 0).
 *   BowVec    TF / TF_IDF: the double sum of w per word in feature order (addWeight); IDF / BINARY: w (addIfNotExist).  Scoring
 *             DOT_PRODUCT needs no normalisation: TF / TF_IDF weights are divided by the number of words, IDF / BINARY kept.
 *             Otherwise BowVector::normalize: L1 = the sum of |w| in ascending word order (L1_NORM, CHI_SQUARE, KL, BHATTACHARYYA),
 *             L2 = sqrt of the sum of w * w in that order (L2_NORM); each weight divided by the norm only if it is > 0.
 * Semantic key j < *n_keep_device is extractor key keep_idx_device[j] (j when NULL) of desc_device.  Outputs, each may be NULL:
 * node_device[j] = the key's mFeatVec node or -1 when the key is in no FeatureVector entry (sivo_keyframe_keys.node's convention);
 * word_device[j] = its BowVector word or -1 likewise (both sivo_orb_capacity(left) room); bow_word_device / bow_weight_device =
 * mBowVec as ascending word ids and double weights (capacity room), *bow_len_device (int64) its length.  The count is clamped to
 * the capacity; a negative count (the -1 of sivo_segnet_semantic_keys_device) writes only *bow_len_device = -1.  A key index
 * outside the capacity gives node and word -1.  The same call computes KeyFrame::ComputeBoW on sivo_keyframe_gather_device's copy
 * (keep_idx NULL).  Runs on `stream` (NULL = the left extractor's stream) with no waits and no host synchronisation; it reads
 * only the vocabulary and its inputs, so LocalMapping's thread may run it concurrently with Tracking's calls on the same extractor.  SIVO_EINVAL for NULL handles or inputs, levelsup < 0, or a
 * vocabulary on another device; SIVO_ERANGE for an extractor capacity above 16,384 keys (the BowVector is sorted in shared memory). */
int sivo_compute_bow_device(const sivo_vocabulary_t* voc, const sivo_orb_t* left, const uint8_t* desc_device, const int* keep_idx_device,
                            const long long* n_keep_device, int levelsup, int* node_device, int* word_device, int* bow_word_device,
                            double* bow_weight_device, long long* bow_len_device, void* stream);
/* Host form: n host descriptors (n x 32); node / word (n), bow_word / bow_weight (n room), *bow_len, any may be NULL.  It stages
 * the descriptors on the vocabulary's device, runs the device form's kernels and synchronises.  SIVO_EINVAL as above and for
 * n < 0; SIVO_ERANGE for n > 16,384. */
int sivo_compute_bow(const sivo_vocabulary_t* voc, const uint8_t* desc, int n, int levelsup, int* node, int* word, int* bow_word,
                     double* bow_weight, int* bow_len);

/* ---- ORBmatcher::SearchByBoW(KeyFrame*, Frame&, vpMapPointMatches) (ORBmatcher.cc:161-284), batched over keyframes: Tracking::
 * TrackReferenceKeyFrame (ratio 0.7, orientation check; Tracking.cc:597-639) and Relocalization's candidates (0.75;
 * Tracking.cc:1237-1286) ---------------------------------------------------------------------------------------------------------
 * Every operation is the IEEE float operation as written.  oracle/bow_oracle.py restates the rules:
 *   walk      nodes present in both FeatureVectors, ascending id; within a node the keyframe's keys in ascending index, only those
 *             with a point (kf_point >= 0); candidates are the frame's keys of that node, ascending index, not yet matched by this
 *             call (vpMapPointMatches starts empty per call).  Best and second-best folded with strict `<` (:209-226); accepted iff
 *             bestDist <= TH_LOW (50) and (float) bestDist < nnratio * (float) bestDist2 (a second best of 256 counts); the accepted
 *             key claims its frame key.
 *   rotation  with check_orientation: rot = kf angle - frame angle, + 360 if negative; bin = roundf(rot * (1.f / 30)), 30 -> 0 (bins
 *             0..12 only, the reference's factor); ComputeThreeMaxima with its 0.1f * max1 rule; every match in another bin is
 *             nulled and the count decremented.
 *   angles    the projection searches' angle rule: key angles finite and in [0, 360].  The host form returns SIVO_ERANGE for any
 *             other frame or keyframe key angle; the device form puts such a frame key in no node and does not search such a
 *             keyframe key.
 * Claims involve only frame keys of one node and each frame key is in one node, so the device runs one warp per (keyframe, common
 * node), walking that node's keyframe keys in order with lanes over the candidates; the histogram is applied after the walk.
 * Frame: semantic key j < *n_keep_device is extractor key keep_idx_device[j] (j when NULL) of kps_device / desc_device, node_device[j]
 * its node (sivo_compute_bow_device's output).  Keyframe k: keyframes[k].kps / desc / node / count (device, sivo_orb_capacity(left)
 * keys; the other members are not read) and kf_point_device[k][i] = the index of GetMapPointMatches()[i] in the caller's
 * sivo_map_point array, -1 for NULL or isBad().  Outputs: match_device[k cap + j] (cap = sivo_orb_capacity(left)) = the point
 * keyframe k's search gave frame key j, or -1 (so sivo_pose_gather_device takes match_device + k cap); n_matches_device[k] (int64)
 * = the function's return.  Counts are clamped to the capacity; a negative count in the frame or in keyframe k writes only
 * n_matches_device[k] = -1 for every affected k.  Runs on `stream` (NULL = the left extractor's stream) with no waits and no host
 * synchronisation.  SIVO_EINVAL for NULL handles, inputs or outputs, n_kf < 0, or nnratio not finite; SIVO_ERANGE for a capacity above 16,384 keys. */
int sivo_search_by_bow_device(const sivo_orb_t* left, const sivo_keypoint* kps_device, const uint8_t* desc_device,
                              const int* keep_idx_device, const long long* n_keep_device, const int* node_device,
                              const sivo_keyframe_keys* keyframes, const int* const* kf_point_device, int n_kf, float nnratio,
                              int check_orientation, int* match_device, long long* n_matches_device, void* stream);
/* Host form: n frame keys gathered per semantic key (mvKeysSemantic, mDescriptorsSemantic, node); keyframes[k]'s kps / desc / node
 * and kf_point[k] host arrays of *keyframes[k].count keys (a negative count: n_matches[k] = -1); match (n_kf x n, row k at k n)
 * and n_matches (n_kf).  It stages the inputs, runs the device form's kernels and synchronises.  SIVO_EINVAL as above and for
 * n < 0; SIVO_ERANGE for an angle that breaks the angle rule and for n above 16,384. */
int sivo_search_by_bow(const sivo_orb_t* left, const sivo_keypoint* kps, const uint8_t* desc, const int* node, int n,
                       const sivo_keyframe_keys* keyframes, const int* const* kf_point, int n_kf, float nnratio, int check_orientation,
                       int* match, long long* n_matches);

/* ---- Tracking::Relocalization's pose hypotheses: PnPsolver (PnPsolver.cc) with SetRansacParameters(0.99, 10, 300, 4, 0.5, 5.991),
 * batched over the candidate keyframes ------------------------------------------------------------------------------------------
 * Every operation is the IEEE float / double operation as written (no contracted multiply-add).  oracle/pnp_oracle.py restates
 * the rule and the reference facts kept; in short:
 *   setup     candidate k's correspondences are the semantic keys j < *n_keep_device in order with 0 <= match[k cap + j] <
 *             n_points (cap = sivo_orb_capacity(left)), a key index inside the capacity and an octave inside the extractor's
 *             levels: mvP2D = the key's (x, y), mvP3Dw = the point's pos, maxError = sigma2[octave] * 5.991f.  N = their number;
 *             minInliers = max((int)(N * 0.5f), 10); epsilon = max(0.5f, (float) minInliers / N); maxIts = 1 when minInliers ==
 *             N, else max(1, min(ceil(log(1 - 0.99) / log(1 - e^3)), 300)) in double with e^3 = (e * e) * e (a NaN or infinite
 *             quotient counts as INT_MIN, so maxIts = 1).  maxIts <= 35 always.
 *   iterate   iterate(n): no pose and no_more at once when N < minInliers.  Otherwise hypotheses g = mnIterations,
 *             mnIterations + 1, ... while mnIterations < maxIts || (this call's count) < n; a hypothesis whose inlier count is
 *             >= minInliers replaces the best set only with a strictly greater count, then Refine runs on the BEST set so far and
 *             returns its pose iff its count > minInliers.  After the loop, mnIterations >= maxIts gives no_more and, when the
 *             best count >= minInliers, the best pose.
 *   draws     hypothesis g's minimal set: Philox4x32-10 (philox.cuh) with ctr = (g, kf_id[k], frame_id lo, frame_id hi), key =
 *             (seed lo, seed hi); draw i (0..3) = int((double) word_i / 2^32 * (N - i)), then the reference's swap-remove.  This
 *             replaces the reference's global rand() stream; every hypothesis is independent of the others.
 *   EPnP      compute_pose (PnPsolver.cc:482-531) in double as written, with every decomposition the documented one-sided Jacobi
 *             rule (jacobi.cuh: pairs in row-major order, rotate while |gamma| > 2^-52 sqrt(alpha beta), at most 30 sweeps;
 *             columns by descending squared norm, ties in column order).  cvSVD's D = the column norms, V = the rotated
 *             identity, U's column = B's column / its norm.  cvSolve / cvInvert(CV_SVD) keep singular value j iff sigma_j >
 *             2^-51 * sum(sigma) (OpenCV's SVBkSb threshold): x = sum_j V_j ((B_j . b) / sigma_j^2).  gauss_newton's x starts
 *             at 0 and qr_solve's early return keeps it.  Sums over correspondences run in correspondence order (Refine's MtM: below).
 *   departs   from cv::SVD: singular vector signs are Jacobi's; a zero singular value of ABt (coplanar or collinear sets) gives a
 *             NaN column of U (0 / 0) where cv::SVD completes a basis, so the hypothesis' pose is NaN and it has no inliers.
 *   inliers   CheckInliers (:318-347): Xc, Yc, invZc rounded to float from double expressions, ue / ve in double, distX / distY
 *             rounded to float, error2 < maxError in float.  Poses are Rcw | tcw rounded to float.
 *   Refine    the same compute_pose over the best set's correspondences, one block per candidate: alphas across threads, MtM in a
 *             fixed tree (thread t of 256 sums correspondences t, t + 256, ... in order; xor shuffles 16 .. 1 in each warp; the 8
 *             warp totals folded by halves), every other sum in correspondence order in one thread.  The reference sums MtM in row
 *             order; the two agree to rounding.
 *   cost      EPnP's decompositions run in one thread per hypothesis and per Refine; k_pnp_hyp and k_pnp_decide use 255 registers
 *             and spill a few hundred bytes (the 12 x 12 and 6 x K working arrays).
 * Handle: one PnPsolver per candidate, kept across calls (mnIterations, the best count, set and pose).  The extractor must outlive
 * the handle.  Calls on one handle must be ordered on one stream. */
typedef struct sivo_pnp sivo_pnp_t;
/* max_candidates in [1, 256]; SIVO_EINVAL otherwise.  Enqueues nothing: the candidates' state is written by setup. */
int sivo_pnp_create(const sivo_orb_t* left, int max_candidates, uint64_t seed, sivo_pnp_t** out);
void sivo_pnp_destroy(sivo_pnp_t* h);
/* Builds n_kf PnPsolvers (n_kf <= max_candidates) from sivo_search_by_bow_device's outputs as they are: match_device (n_kf rows of
 * cap ints), n_matches_device (n_kf int64).  Frame keys as for the other Frame-tail calls (keep_idx_device NULL = identity);
 * points_device the map points the rows index.  kf_id (host, n_kf) and frame_id select the draws.  A negative frame count or
 * n_matches_device[k] makes candidate k return no_more with no pose.  Resets every candidate's state.  Runs on `stream` (NULL = the
 * left extractor's stream) with no host synchronisation; the inputs may be reused once it has run.  SIVO_EINVAL for NULL handles
 * or inputs, n_kf outside [0, max_candidates], n_points < 0 or a camera parameter not finite. */
int sivo_pnp_setup_device(sivo_pnp_t* h, const sivo_keypoint* kps_device, const int* keep_idx_device, const long long* n_keep_device,
                          const int* match_device, const long long* n_matches_device, const sivo_map_point* points_device,
                          int n_points, const uint32_t* kf_id, int n_kf, uint64_t frame_id, float fx, float fy, float cx, float cy,
                          void* stream);
/* iterate(n_iterations) on every candidate k of the last setup with active[k] != 0 (host array; the others are neither run nor
 * written).  Per active k: Tcw_device[12 k ..] (3 x 4 row-major, usable as sivo_pose_optimize_device's Tcw_in) when
 * has_pose_device[k]; no_more_device[k]; n_inliers_device[k]; inlier_match_device[k cap + j] = match[k cap + j] for the
 * inliers, -1 for every other j < cap (the row that becomes mvpMapPoints).  SIVO_EINVAL for NULL handles or outputs. */
int sivo_pnp_iterate_device(sivo_pnp_t* h, int n_iterations, const uint8_t* active, float* Tcw_device, int* has_pose_device,
                            int* no_more_device, int* inlier_match_device, int* n_inliers_device, void* stream);
/* Test hooks.  sivo_dbg_pnp_state synchronises the device, then per candidate of the last setup: out[7 k ..] = N, minInliers,
 * maxIts, mnIterations, best count, the best set's Refine has failed, dead (a negative count); eps[k] = epsilon (may be NULL). */
int sivo_dbg_pnp_state(const sivo_pnp_t* h, int* out, float* eps);
typedef struct sivo_pnp_pose_debug {
  double cws[12];                          /* control points, 4 x 3 */
  double d[12], ut[144];                   /* MtM's singular values (descending); Ut: row r = V's column for d[r] */
  double l_6x10[60], rho[6];
  double betas[12];                        /* approximations 1, 2, 3 after gauss_newton, 4 each */
  double Rs[27], ts[9], rep_errors[3];     /* compute_R_and_t of each */
  double R[9], t[3];                       /* the chosen one */
  int32_t best, reserved;                  /* 1, 2 or 3 */
} sivo_pnp_pose_debug;
/* Refine's kernel path (block_pose: the gather, compute_pose with MtM in its tree order, CheckInliers) on n >= 1 host
 * correspondences, all selected: p3d n x 3, p2d n x 2, max_err n (floats).  Outputs alphas (4 n, may be NULL), mask ((n + 31) / 32
 * words, may be NULL), *n_inliers (may be NULL) and *dbg. */
int sivo_dbg_pnp_compute_pose(int device, const float* p3d, const float* p2d, const float* max_err, int n, float fx, float fy, float cx,
                              float cy, double* alphas, uint32_t* mask, int* n_inliers, sivo_pnp_pose_debug* dbg);
/* k_pnp_hyp itself for candidate k of the last setup, hypotheses first .. first + n_hyp - 1, without touching the state (it
 * synchronises the device): draws[4 h ..], Rt[12 h ..] (R row-major, then t, doubles), counts[h] (-1 when the candidate has no
 * hypotheses: dead or N < minInliers), masks[h words ..] (words = (sivo_orb_capacity + 31) / 32). */
int sivo_dbg_pnp_hypotheses(sivo_pnp_t* h, int k, int first, int n_hyp, int* draws, double* Rt, int* counts, uint32_t* masks);
/* The minimal sets of hypotheses first .. first + n_hyp - 1 among N >= 4 correspondences: out[4 h ..]. */
int sivo_dbg_pnp_draws(int device, uint64_t seed, uint32_t kf_id, uint64_t frame_id, int first, int n_hyp, int N, int* out);

/* Best / second-best match over per-query candidate lists -- the inner loop of ORBmatcher::SearchByProjection
 * (ORBmatcher.cc:79-113), its last-frame / keyframe variants (:1278-, :1420-), SearchForTriangulation (:631-) and
 * SearchBySim3 (next row 4).  Query i's candidates are cand_idx[cand_offsets[i] .. cand_offsets[i+1]) (indices into the
 * train descriptors, in the order GetFeaturesInArea returned them; the caller has already dropped the ones its own
 * state excludes).  out5[5 i ..] = {bestIdx, bestDist, bestLevel, bestDist2, bestLevel2} exactly as the sequential loop
 * leaves them (strict '<', so the first minimum wins; 256 / -1 when there is no candidate).  train_level (octave per train
 * keypoint) may be NULL (levels reported as 0).  The TH_HIGH / mfNNratio / orientation-histogram decisions stay with the
 * caller, as does the in-loop `F.mvpMapPoints[bestIdx] = pMP` dependency between queries. */
int sivo_hamming_best2(int device, const uint8_t* query_desc, int n_query, const uint8_t* train_desc, int n_train,
                       const int* cand_offsets, const int* cand_idx, const int* train_level, int* out5);

/* ---- test hooks for single layers (float NCHW host arrays in/out; run the product kernels) ----- */
int sivo_dbg_pool(int device, const float* in, int n, int c, int h, int w, float* out, int* mask);
int sivo_dbg_unpool(int device, const float* in, const int* mask, int n, int c, int h, int w, float* out);
int sivo_dbg_conv(int device, int engine, int precision, const float* in, int n, int cin, int h, int w,
                  const float* weight, const float* bias, const float* bn_scale, const float* bn_shift,
                  int cout, int k, int pad, int relu, float* out);
/* The 7x7 float-logits convolution over the max-unpool of `pooled` (float NCHW [n][64][h][w]) by `mask` (sivo_dbg_unpool's
 * convention, [mask_n][64][h][w], image i takes mask i % mask_n), unpooled as the kernel loads its input rows: out = float
 * NCHW [n][cout][2h][2w], cout <= 16, k = 7, no ReLU.  Equals sivo_dbg_unpool followed by sivo_dbg_conv bit for bit. */
int sivo_dbg_conv_unpooled(int device, const float* pooled, const int* mask, int n, int mask_n, int h, int w, const float* weight,
                           const float* bias, const float* bn_scale, const float* bn_shift, int cout, int k, float* out);
/* The 7x7 64 -> 64 half convolution (Basic's decoder layers: bias, no ReLU) over the max-unpool of `pooled` by `mask`
 * (conventions as above): out = float NCHW [n][64][2h][2w].  drop_layer >= 0: the sampling dropout of that layer (seed,
 * frame; image i is sample i, scale 2) is applied in its epilogue.  unpool_on_load = 1: the kernel expands the pooled input
 * as it loads its input rows; 0: the unpool kernel writes the unpooled tensor and the same convolution reads it.  The two
 * are equal bit for bit. */
int sivo_dbg_conv64_unpooled(int device, const float* pooled, const int* mask, int n, int mask_n, int h, int w, const float* weight,
                             const float* bias, int drop_layer, uint64_t seed, uint64_t frame, int unpool_on_load, float* out);
int sivo_dbg_lrn(int device, const float* in, int n, int c, int h, int w, int size, float alpha, float beta,
                 float k, float* out);
int sivo_dbg_mc_reduce(int device, const float* logits, int T, int c, int h, int w, uint8_t* classes,
                       double* confidence, double* entropy);
/* logits float NCHW [T][c][h][w] (T >= 2) laid out as sivo_dbg_mc_reduce does (c <= 16: the 16-channel layout and the quad
 * kernel; c > 16: the generic kernel); classes / variance h x w. */
int sivo_dbg_mc_variance(int device, const float* logits, int T, int c, int h, int w, const uint8_t* classes, double* variance);
int sivo_dbg_dropout_mask(int device, uint64_t seed, uint64_t frame, int layer, int T, int c, int h, int w,
                          uint8_t* keep);

const char* sivo_last_error(void);
const char* sivo_version(void);

#ifdef __cplusplus
}
#endif
#endif /* SIVO_B200_H_ */
