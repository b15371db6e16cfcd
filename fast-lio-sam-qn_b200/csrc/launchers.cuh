// launchers.cuh -- host entry points of the kernel files.  Both the file that defines a launcher and every file that calls
// it include this header, so a signature that drifts fails the build instead of the load.
#pragma once
#include <cstddef>

#include "internal.cuh"

namespace b200 {

// index_build.cu
size_t radix_sort_ws_bytes(int n, int key_bits);
int radix_sort_result_buf(int key_bits);
int launch_radix_sort(const CloudDev* d_clouds, int count, int max_n, int key_bits, cudaStream_t s);
int launch_index_build(const CloudDev* d_clouds, int count, int max_n, cudaStream_t s);

// gicp.cu.  launch_covariances: k <= 32 one thread per point; k > 32 goes to launch_covariance_large and needs
// covariance_large_slab_bytes(count, max_n, k) of device scratch in slab (nullptr when that is 0)
int launch_covariances(const CloudDev* d_clouds, int count, int max_n, int k, int method, unsigned long long* slab, cudaStream_t s);
void launch_gicp_init(const PairDev* pairs, PairState* states, const double* d_guess, LmCall* call, LmSched* sched, cudaStream_t s);
// n_cached: slot entries the step kernels cache in shared memory, lm_slot_cache(capacity of the LM arena)
void launch_gicp_search(const PairDev* pairs, const PairState* states, int blocks, const LmCall* call, const LmSched* sched, int n_cached,
                        cudaStream_t s);
void launch_gicp_accum(const PairDev* pairs, const PairState* states, int blocks, const LmSched* sched, int n_cached, cudaStream_t s);
void launch_gicp_control(const PairDev* pairs, PairState* states, LmCall* call, LmSched* sched, cudaStream_t s);
cudaError_t lm_graph_build(LmGraph* g, const PairDev* pairs, PairState* states, const double* guess, LmCall* call, LmSched* sched,
                           int blocks_search, int blocks_accum, int n_cached);
void lm_graph_destroy(LmGraph* g);
int launch_knn_queries(const CloudDev& c, const float* d_q, int nq, int qstride, int k, int* idx, float* d2, cudaStream_t s, int brute);
void launch_set_covariances(const CloudDev& c, const double* d_cov9, cudaStream_t s);
int launch_lm_step_tap(const b200reg_lm_case* d_cases, int n, b200reg_lm_step* d_out, cudaStream_t s);
void launch_transform_out(const CloudDev& c, const float* d_Tf, float* d_out3, cudaStream_t s);

// quatro.cu
cudaError_t quatro_init_device();
int launch_fpfh(const CloudDev* d_clouds, int count, int max_n, float normal_r2, float fpfh_r2, cudaStream_t s);
// the stages of launch_fpfh and launch_quatro_match_solve that b200reg_match_tap runs on caller descriptors:
//   launch_load_records   rows of 33 bins in c.fpfh (stride FPAD) -> records, original index = row (the k_fpfh tail)
//   launch_feature_order  k_fcode, radix sort, k_fgather (keys / vals / hist as for launch_radix_sort)
//   launch_feature_match  k_match_init, k_feat_nn both ways, k_first_hit, k_mutual
int launch_load_records(const CloudDev* d_clouds, int count, int max_n, cudaStream_t s);
int launch_feature_order(const CloudDev* d_clouds, int count, int max_n, cudaStream_t s);
int launch_feature_match(const MatchDev* d_pairs, int count, int max_ni, int max_nj, float thr2, int advanced, cudaStream_t s);
// optimizedMatching: k_teaser_solve solves the sets of at most MAXC and leaves larger ones (counters[2] > MAXC) to
// launch_big_solve
int launch_quatro_match_solve(const MatchDev* d_pairs, int count, int max_ni, int max_nj, const QuatroParamsDev& prm, cudaStream_t s);
// k_teaser_solve alone (one block of solve_smem_bytes() per pair): counters[2] correspondences listed in out_corr
size_t solve_smem_bytes();
int launch_teaser_solve(const MatchDev* d_pairs, int count, const QuatroParamsDev& prm, cudaStream_t s);
// k_big_gather + launch_big_graph_solve(n_wide = 0): pairs of at most max_n <= BIGC correspondences, `big` bound
int launch_big_solve(const MatchDev* d_pairs, int count, int max_n, const QuatroParamsDev& prm, cudaStream_t s);
int launch_adv_wide(const MatchDev* d_pair, int n, const QuatroParamsDev& prm, cudaStream_t s);
int launch_big_graph_solve(const MatchDev* d_pairs, int count, const QuatroParamsDev& prm, int n_wide, cudaStream_t s);
void launch_transform_raw(const CloudDev* d_clouds, const double* d_T16s, int count, int max_n, float4* const* d_outs, cudaStream_t s);

// radius.cu: the stages of b200reg_radius_search (order, count, scan, fill, segmented sort); each returns its launches
int launch_radius_query_keys(const CloudDev& c, const float* d_q, int nq, int qstride, uint32_t* keys, uint32_t* vals, cudaStream_t s);
int launch_radius_count(const CloudDev& c, const float* d_q, int qstride, const uint32_t* order, int nq, float r2, int* counts,
                        cudaStream_t s);
size_t radius_scan_ws_bytes(int nq);
int launch_radius_scan(const int* counts, int nq, int64_t* offsets, void* ws, cudaStream_t s);
int launch_radius_chunk_keys(const uint32_t* order, int nq, const int* starts, int nchunks, uint32_t* keys, uint32_t* vals,
                             cudaStream_t s);
struct RadiusChunk {  // one chunk of queries: sorted rows [r0, r0 + nr) of `order`, caller indices [q0, q0 + nr)
  int r0, nr, q0;
  int64_t base;     // offsets[q0]: entry e of the chunk is neighbour (base + e) of the whole call
  int* e_idx;       // [entries] original point index
  float* e_d2;      // [entries]
  uint32_t* e_seg;  // [entries] caller index - q0
  uint32_t* keys;   // [entries] sort input: the original index ...
  uint32_t* vals;   // [entries] ... and the entry itself
};
int launch_radius_fill(const CloudDev& c, const float* d_q, int qstride, const uint32_t* order, float r2, const int64_t* offsets,
                       const RadiusChunk& ch, cudaStream_t s);
int launch_radius_rekey(const uint32_t* perm, int m, const uint32_t* src, uint32_t* keys, cudaStream_t s);
int launch_radius_gather(const uint32_t* perm, int m, const int* e_idx, const float* e_d2, int* idx_out, float* d2_out, cudaStream_t s);

// knn_large.cu: exact k-NN for k > 32, one warp per query.  Lists of up to KL_SMEM_K entries live in shared memory; longer
// ones need slab = nq * k keys of device scratch (unused otherwise)
constexpr int KL_SMEM_K = 256;
int launch_knn_large(const CloudDev& c, const float* d_q, int nq, int qstride, int k, unsigned long long* slab, int* idx, float* d2,
                     cudaStream_t s);
// Covariances for k > 32, one warp per point, every cloud of the call in one launch.  A warp's neighbour list holds
// min(k, max_n) keys; lists longer than KL_SMEM_K live in a slab with one list per warp of the grid, not per point, so the
// launcher caps the grid to keep the slab at or below max(KL_COV_SLAB_BYTES, one 4-warp block's lists = 32 * min(k, max_n)
// bytes) whatever the cloud sizes.  covariance_large_slab_bytes is that slab's exact size (0 for the shared-memory tier).
constexpr size_t KL_COV_SLAB_BYTES = size_t(128) << 20;
size_t covariance_large_slab_bytes(int count, int max_n, int k);
int launch_covariance_large(const CloudDev* d_clouds, int count, int max_n, int k, int method, unsigned long long* slab,
                            cudaStream_t s);

// assemble.cu
void launch_pack_xyzi(const float* d_raw, int stride, int n, float4* d_out, cudaStream_t s);
void launch_ingest_world(const float* d_raw, int stride, int n, const double* d_Tinv, float4* d_out, cudaStream_t s);
int launch_fetch_closest(const double* d_pos, const double* d_stamp, const int* d_queries, int count, double radius, double tdiff,
                         int* d_out, cudaStream_t s);
int launch_assemble_voxelize(const AssembleJob* d_jobs, const CloudDev* d_sort, int count, int max_total, const KeyframeDev* d_kfs,
                             const double* d_poses, float inv_leaf, cudaStream_t s);
// loop-cloud capture: intensities of freshly uploaded clouds (raw records still valid) into d_inten[i][n_i]; then every
// CaptureRow of a call (max_n = the longest row)
void launch_gather_intensity(const CloudDev* d_clouds, int count, int max_n, float* const* d_inten, cudaStream_t s);
void launch_capture_rows(const CaptureRow* d_rows, int nrows, int max_n, cudaStream_t s);

}  // namespace b200
