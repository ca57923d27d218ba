// The Frame-tail stages behind the C ABI (capi.cu): stereo and Hamming matching (stereo.cu), information selection (info.cu),
// projection searches and the keyframe Fuse (track.cu) and pose optimisation (pose.cu).  A name ending in _device works on device-resident arrays and
// enqueues on a stream without a host synchronisation; the others take host arrays and return with the results downloaded.
// Each function's contract is written above its definition.
#pragma once
#include "orb.h"

namespace sivo {

// ---- stereo.cu
void stereo_hamming(int device, const sivo_keypoint* left, const uint8_t* dl, int nl, const sivo_keypoint* right,
                    const uint8_t* dr, int nr, const float* scale, int nlevels, int rows, float min_d, float max_d,
                    int* best_idx, int* best_dist);
void hamming_best2(int device, const uint8_t* query, int nq, const uint8_t* train, int nt, const int* cand_off, const int* cand_idx,
                   const int* train_level, int* out5);
void stereo_match(const Orb& left, const Orb& right, const sivo_keypoint* kl, const uint8_t* dl, int nl, const sivo_keypoint* kr,
                  const uint8_t* dr, int nr, float mb, float mbf, float* u_right, float* depth);
void stereo_match_device(Orb& left, Orb& right, const sivo_keypoint* kl, const uint8_t* dl, const int* keep_idx, const long long* n_left,
                         const sivo_keypoint* kr, const uint8_t* dr, const long long* n_right, float mb, float mbf, float* u_right,
                         float* depth, cudaStream_t s);
void stereo_median_cut(int device, const int* sad, int n, float* u, float* z);

// ---- info.cu
void info_select(const Orb& left, const sivo_keypoint* kps, const float* depth, const double* entropy, int n, const sivo_info_camera& cam,
                 double threshold, float* world, double* reduction, int* selected, int* n_selected);
void info_terms(const Orb& left, const sivo_keypoint* kps, const float* depth, int n, const sivo_info_camera& cam, float* world,
                double* det_state, double* det_meas, double* det_joint);
void info_select_device(const Orb& left, const sivo_keypoint* kps, const double* kp_entropy, const int* keep_idx, const long long* n_keep,
                        const float* depth, const sivo_info_camera& cam, double threshold, float* world, double* reduction, int* selected,
                        long long* n_selected, cudaStream_t s);

// ---- track.cu
void search_local_points(const Orb& left, const sivo_keypoint* kps, const uint8_t* desc, const float* u_right, const uint8_t* blocked, int n,
                         const sivo_map_point* pts, int n_points, const sivo_track_frame& f, float th, float nnratio, uint8_t* in_view,
                         int* match, int* n_matches);
void search_last_frame(const Orb& left, const sivo_keypoint* kps, const uint8_t* desc, const float* u_right, int n, const sivo_map_point* pts,
                       int n_points, const sivo_track_frame& f, const float* Rlw, const float* tlw, float th, int* match, int* n_matches);
void search_local_points_device(const Orb& left, const sivo_keypoint* kps, const uint8_t* desc, const int* keep_idx, const long long* n_keep,
                                const float* u_right, const uint8_t* blocked, const sivo_map_point* pts, int n_points,
                                const sivo_track_frame& f, float th, float nnratio, uint8_t* in_view, int* match, long long* n_matches,
                                cudaStream_t s);
void search_last_frame_device(const Orb& left, const sivo_keypoint* kps, const uint8_t* desc, const int* keep_idx, const long long* n_keep,
                              const float* u_right, const sivo_map_point* pts, int n_points, const sivo_track_frame& f, const float* Rlw,
                              const float* tlw, float th, int* match, long long* n_matches, cudaStream_t s);
void features_in_area(const Orb& left, const sivo_keypoint* kps, int n, const sivo_track_frame& f, const float* xyr, const int* levels, int nq,
                      int* offsets, int* idx, int idx_cap);
void fuse_device(const Orb& left, const sivo_keyframe_keys* targets, int n_targets, const sivo_fuse_camera& cam, const sivo_map_point* pts,
                 int n_points, float th, int* match, int* dist, cudaStream_t s);
void fuse_host(const Orb& left, const sivo_keyframe_keys* targets, int n_targets, const sivo_fuse_camera& cam, const sivo_map_point* pts,
               int n_points, float th, int* match, int* dist, int* stage);

// ---- pose.cu
void pose_optimize_device(const Orb& left, const sivo_keypoint* kps, const int* keep_idx, const long long* n_keep, const float* u_right,
                          const float* xw, float fx, float fy, float cx, float cy, float mbf, const float* Tcw_in,
                          sivo_pose_result* result, uint8_t* outlier, cudaStream_t s);
void pose_gather_device(const Orb& left, const int* match, const long long* n_keep, const sivo_map_point* pts, int n_points, float* xw,
                        cudaStream_t s);
void pose_optimize(const Orb& left, const sivo_keypoint* kps, const float* u_right, const float* xw, int n, float fx, float fy, float cx,
                   float cy, float mbf, const float* Tcw_in, sivo_pose_result* result, uint8_t* outlier);
int pose_trace(const Orb& left, const sivo_keypoint* kps, const float* u_right, const float* xw, int n, float fx, float fy, float cx,
               float cy, float mbf, const float* Tcw_in, sivo_pose_result* result, uint8_t* outlier, sivo_pose_trace_rec* trace,
               int trace_cap);
void pose_se3(int device, int n, const float* T, const double* d, double* se3, double* up, double* tv, sivo_pose_result* res);
void pose_system(const Orb& left, const sivo_keypoint* kps, const float* u_right, const float* xw, int n, float fx, float fy, float cx,
                 float cy, float mbf, const double* pose7, int robust_stereo, const uint8_t* level1, double* err, double* chi2, double* rho,
                 double* jac, double* H, double* b, double* chi);

// ---- mapping.cu
void keyframe_gather_device(const Orb& left, const sivo_keypoint* kps, const uint8_t* desc, const int* keep_idx, const long long* n_keep,
                            const float* u_right, const float* depth, const uint8_t* cls, const double* conf, const double* ent,
                            sivo_keypoint* o_kps, uint8_t* o_desc, float* o_ur, float* o_depth, uint8_t* o_cls, double* o_conf,
                            double* o_ent, long long* o_count, cudaStream_t s);
void create_map_points_device(const Orb& left, const sivo_keyframe_keys& kf1, const sivo_keyframe_keys* nbs, int n_nb,
                              const sivo_mapping_params& prm, int* created_nb, int* created_idx, float* world, int* created_list,
                              long long* n_created, cudaStream_t s);
void create_map_points_host(const Orb& left, const sivo_keyframe_keys& kf1, const sivo_keyframe_keys* nbs, int n_nb,
                            const sivo_mapping_params& prm, int* dbg_match, int* dbg_stage, double* dbg_red, int* created_nb,
                            int* created_idx, float* world, int* created_list, long long* n_created);

// ---- pnp.cu
constexpr int kPnpMaxCandidates = 256;
struct Pnp;
Pnp* pnp_create(const Orb& left, int max_candidates, uint64_t seed);
void pnp_destroy(Pnp* h);
void pnp_setup_device(Pnp& h, const sivo_keypoint* kps, const int* keep_idx, const long long* n_keep, const int* match,
                      const long long* n_matches, const sivo_map_point* points, int n_points, const uint32_t* kf_id, int n_kf,
                      uint64_t frame_id, float fx, float fy, float cx, float cy, cudaStream_t s);
void pnp_iterate_device(Pnp& h, int n_iterations, const uint8_t* active, float* Tcw, int* has_pose, int* no_more, int* inlier_match,
                        int* n_inliers, cudaStream_t s);
void pnp_state(const Pnp& h, int* out, float* eps);
void pnp_compute_pose_debug(int device, const float* p3d, const float* p2d, const float* max_err, int n, float fx, float fy, float cx,
                            float cy, double* alphas, uint32_t* mask, int* n_inliers, sivo_pnp_pose_debug* dbg);
void pnp_hypotheses(Pnp& h, int k, int first, int n_hyp, int* draws, double* Rt, int* counts, uint32_t* masks);
void pnp_draws(int device, uint64_t seed, uint32_t kf_id, uint64_t frame_id, int first, int n_hyp, int N, int* out);

}  // namespace sivo
