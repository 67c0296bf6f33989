/* dliom_b200 — C-ABI of the H100-native (sm_90a) scan-registration hot path.
 *
 * Every entry point replaces one CPU interface of the reference (peterWon/D-LIOM, a Cartographer fork).
 * Citations: C/ = src/cartographer/cartographer/, SM/ = C/mapping/internal/3d/scan_matching/,
 * LTB = C/mapping/internal/3d/local_trajectory_builder_3d.cc.
 *
 * Conventions
 *   - plain pointers and sizes only; all buffers are caller-owned HOST memory unless the name ends in _dev;
 *   - a pose is 7 doubles: t.x t.y t.z q.w q.x q.y q.z (the reference's CeresPose order, ceres_pose.cc:23-28);
 *   - a point cloud is n rows of `stride` floats, the first three being x y z
 *     (stride 3 = sensor::PointCloud, 4 = TimedPointCloud, 8 = RangeMeasurement{Vector4f,size_t});
 *   - every function returns DL_OK (0) or a negative dl_status; nothing aborts (the reference CHECK-fails,
 *     SM/ceres_scan_matcher_3d.cc:89-92); dl_last_error() gives the message for the calling context;
 *   - a dl_context owns one CUDA stream plus scratch and must be used by one host thread at a time;
 *     create one per thread for the re-entrant use ConstraintBuilder3D makes of CeresScanMatcher3D::Match
 *     (C/mapping/internal/constraints/constraint_builder_3d.cc:318-326). dl_grid objects are shared, read-only
 *     during matching.
 *   - there is no CPU fallback: without a CUDA device every call fails with DL_ERR_CUDA.
 */
#ifndef DLIOM_B200_H_
#define DLIOM_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum dl_status {
  DL_OK = 0,
  DL_ERR_CUDA = -1,        /* CUDA runtime error (incl. no device)                                  */
  DL_ERR_ARG = -2,         /* null pointer, negative size, weight count mismatch, ...               */
  DL_ERR_GRID_RANGE = -3,  /* cell index outside +-8192 cells (hybrid_grid.h:391 CHECK_LE(bits,8)) */
  DL_ERR_EMPTY = -4,       /* empty cloud where the reference would drop the scan (LTB:497-534)     */
  DL_ERR_SCORE = -5        /* RT-CSM best score <= 0 (real_time_correlative_scan_matcher_3d.cc:111) */
} dl_status;

typedef struct dl_context dl_context;
typedef struct dl_grid dl_grid;

int dl_context_create(int device_ordinal, dl_context** out);
void dl_context_destroy(dl_context* ctx);
const char* dl_last_error(const dl_context* ctx);
const char* dl_status_string(int status);
/* Number of kernels this context has launched since creation (bench.py's gpu_launches). */
int64_t dl_context_kernel_launches(const dl_context* ctx);
/* Per-stage device timing of the front end (CUDA events on the context's stream). When enabled, every
 * dl_frontend_* call brackets its stages with events; dl_context_read_profile synchronises, returns the
 * accumulated milliseconds and call counts per stage since the last read, and resets them. */
typedef struct dl_stage_time {
  char name[32];
  double ms;
  int64_t calls;
} dl_stage_time;
int dl_context_set_profiling(dl_context* ctx, int enabled);
/* Host waits of this context sleep (cudaEventBlockingSync) instead of spinning: for the background threads that run loop
 * closure / the pose graph (the reference's thread pool at nice(10), C/common/thread_pool.cc) on hosts with few CPUs. */
int dl_context_set_blocking_sync(dl_context* ctx, int enabled);
int dl_context_read_profile(dl_context* ctx, dl_stage_time* out, int32_t capacity, int32_t* num_stages);
/* The context's cudaStream_t as an integer, and a blocking wait on it. */
uint64_t dl_context_stream(const dl_context* ctx);
int dl_context_synchronize(dl_context* ctx);

/* ---- probability grid: device mirror of mapping::HybridGrid (C/mapping/3d/hybrid_grid.h:411-547) ---------
 * Cells are given as the HybridGrid proto layout (parallel x/y/z/value arrays, hybrid_grid.h:530-542) and must
 * hold post-FinishUpdate values (< 32768). dl_grid_set_cells may be called again after every host
 * InsertRangeData with just the touched cells; only dirty 8^3 bricks are re-uploaded by dl_grid_sync.
 * Sharing: any number of contexts (host threads) may READ a grid concurrently (matchers, loop-closure searches; the search index
 * of a grid is built once under a lock) — as the reference shares a finished Submap3D's HybridGrid between its thread-pool
 * workers. A grid that is being modified (dl_grid_set_cells / dl_grid_sync / dl_*_insert_range_data) must not be in use by
 * another context at the same time: the active submaps belong to the one front-end thread (Node::mutex_ in the reference). */
int dl_grid_create(dl_context* ctx, float resolution, dl_grid** out);
void dl_grid_destroy(dl_grid* grid);
int dl_grid_set_cells(dl_grid* grid, int64_t n, const int32_t* x, const int32_t* y, const int32_t* z,
                      const uint16_t* value);
int dl_grid_sync(dl_grid* grid);
float dl_grid_resolution(const dl_grid* grid);
/* The 8^3 bricks in use: every brick the reference's HybridGrid would have allocated, set or inserted. After a device insert
 * this is the device's count (one 4-byte read-back; -1 on a CUDA error), until an export or dl_grid_set_cells brings the
 * host mirror up to date. */
int64_t dl_grid_num_bricks(const dl_grid* grid);
/* HybridGrid::value() for n cell indices (xyz interleaved), evaluated ON THE DEVICE (hybrid_grid.h:263-281). */
int dl_grid_lookup(dl_context* ctx, const dl_grid* grid, int64_t n, const int32_t* xyz, uint16_t* value_out);
/* InterpolatedGrid::GetProbability (SM/interpolated_grid.h:50-103) and its spatial gradient for n points
 * (xyz interleaved doubles), on the device. out: n rows of 4 doubles (value, d/dx, d/dy, d/dz). */
int dl_grid_interpolate(dl_context* ctx, const dl_grid* grid, int64_t n, const double* xyz, double* out);

/* ---- grid WRITE side (SURVEY 8f-1): RangeDataInserter3D::Insert (C/mapping/3d/range_data_inserter_3d.cc:76-92, misses
 *      :27-51), HybridGrid::ApplyLookupTable / FinishUpdate (hybrid_grid.h:494-520) and Submap3D::InsertRangeData
 *      (C/mapping/3d/submap_3d.cc:264-279) executed ON the device grid, which then is the primary copy (no per-scan host
 *      insert + upload). Options = proto::RangeDataInserterOptions3D. ------------------------------------------------- */
typedef struct dl_range_data_inserter_options {
  double hit_probability;
  double miss_probability;
  int32_t num_free_space_voxels;
  int32_t reserved;
} dl_range_data_inserter_options;
/* returns: n x 3 floats already in the grid's (submap) frame; origin: 3 floats in the same frame.
 * The grid grows to hold exactly the cells the Insert touches: each hit cell and the last num_free_space_voxels samples of
 * its ray. The origin cell counts only when it is one of those samples, so the origin may lie beyond +-8192 cells.
 * Refused before any grid changes (the reference CHECK-fails instead):
 *   DL_ERR_ARG         a ray of 2^15 cells or more (num_samples, the largest |hit cell - origin cell| component), whatever
 *                      num_free_space_voxels is (CHECK_LT(num_samples, 1 << 15), range_data_inserter_3d.cc:37);
 *   DL_ERR_GRID_RANGE  a touched cell outside +-8192 cells.
 * The submap and batched forms check every job of the call before the first one writes. */
int dl_grid_insert_range_data(dl_context* ctx, dl_grid* grid, const dl_range_data_inserter_options* options,
                              const float* origin, const float* returns, int64_t n);
/* Submap3D::InsertRangeData: range data in the LOCAL frame is moved into the submap frame (local_pose^-1, float), the
 * high-resolution grid receives the returns within high_resolution_max_range of the origin, the low-resolution grid all. */
int dl_submap_insert_range_data(dl_context* ctx, dl_grid* high_resolution_grid, dl_grid* low_resolution_grid,
                                const dl_range_data_inserter_options* options, const double* submap_local_pose,
                                int32_t high_resolution_max_range, const float* origin, const float* returns, int64_t n);
/* HybridGrid iteration (the ToProto order, hybrid_grid.h:530-542) of the grid's CURRENT content, downloading the
 * device copy first if it is ahead of the host mirror. Call with capacity 0 to query *n_cells. */
int dl_grid_export_cells(dl_grid* grid, int64_t capacity, int32_t* x, int32_t* y, int32_t* z, uint16_t* value,
                         int64_t* n_cells);

/* ---- sensor::VoxelFilter::Filter (C/sensor/internal/voxel_filter.h:34-62, voxel_filter.cc:81-131) ------------
 * keep_out receives the input-order indices of the first point in each voxel (capacity n). */
int dl_voxel_filter(dl_context* ctx, const float* points, int64_t n, int stride, float resolution,
                    int64_t* keep_out, int64_t* n_keep);
/* Voxel indices only (GetCellIndex, voxel_filter.cc:126-131): out = n rows of 3 int32. */
int dl_voxel_indices(dl_context* ctx, const float* points, int64_t n, int stride, float resolution, int32_t* out);

/* ---- sensor::AdaptiveVoxelFilter::Filter (voxel_filter.cc:28-77,147-150; options proto
 *      C/sensor/proto/adaptive_voxel_filter_options.proto) ------------------------------------------------------ */
typedef struct dl_adaptive_voxel_filter_options {
  float max_length;
  float min_num_points;
  float max_range;
} dl_adaptive_voxel_filter_options;
/* passes_out (optional, capacity 32) receives every voxel edge tried, in order. */
int dl_adaptive_voxel_filter(dl_context* ctx, const dl_adaptive_voxel_filter_options* options, const float* points,
                             int64_t n, int stride, int64_t* keep_out, int64_t* n_keep, float* passes_out,
                             int* n_passes);

/* ---- scan_matching::RealTimeCorrelativeScanMatcher3D::Match
 *      (SM/real_time_correlative_scan_matcher_3d.h:33-60, .cc:34-113; options
 *      C/mapping/proto/scan_matching/real_time_correlative_scan_matcher_options.proto) ------------------------- */
typedef struct dl_rtcsm_options {
  double linear_search_window;
  double angular_search_window;
  double translation_delta_cost_weight;
  double rotation_delta_cost_weight;
} dl_rtcsm_options;
typedef struct dl_rtcsm_info {
  int64_t best_index;    /* linear candidate index in the reference's loop order (z,y,x,rz,ry,rx) */
  int64_t num_candidates;
  int32_t linear_window; /* cells */
  int32_t angular_window;
  float angular_step;
  float max_scan_range;
} dl_rtcsm_info;
/* Returns the best score through score_out (the reference's return value). all_scores (optional) has room for
 * every candidate. */
int dl_rtcsm_match(dl_context* ctx, const dl_rtcsm_options* options, const double* initial_pose,
                   const float* points, int64_t n, const dl_grid* grid, double* pose_out, float* score_out,
                   dl_rtcsm_info* info, float* all_scores);

/* ---- scan_matching::FastCorrelativeScanMatcher3D::MatchWith3DofInitial (SM/fast_correlative_scan_matcher_3d.h:110-160,
 *      .cc:165-196): the loop-closure coarse matcher as this fork calls it (constraint_builder_3d.cc:275-277). The whole
 *      (x, y, z) window is scored on the device; no precomputation grid stack is built (options' depths are accepted and
 *      ignored). Options = proto::FastCorrelativeScanMatcherOptions3D. ------------------------------------------------ */
typedef struct dl_fcsm_options {
  int32_t branch_and_bound_depth;
  int32_t full_resolution_depth;
  double min_rotational_score;
  double min_low_resolution_score;
  double linear_xy_search_window;
  double linear_z_search_window;
  double angular_search_window;
} dl_fcsm_options;
typedef struct dl_fcsm_result { /* FastCorrelativeScanMatcher3D::Result; found == 0 <=> the reference returns nullptr */
  int32_t found;
  float score;
  double pose_estimate[7];
  float rotational_score;
  float low_resolution_score;
  int32_t offset[3];      /* winning translation in cells */
  int32_t scan_index;     /* dl_fcsm_match: which of the yaw steps that passed the rotational score won (0 otherwise) */
  int64_t num_candidates; /* leaves scored */
} dl_fcsm_result;
/* all_scores (optional) receives the score of every leaf, index (z * side + y) * side + x, offsets counted from the window's
 * low corner, and asking for it runs the exhaustive search. With wxy = lround(linear_xy_search_window / (double)resolution),
 * wz = lround(linear_z_search_window / (double)resolution) and side = 2 * wxy + 1 there are num_candidates =
 * side * side * (2 * wz + 1) leaves; an all_scores_capacity (in floats) below that fails with DL_ERR_ARG before any work. */
int dl_fcsm_match_3dof(dl_context* ctx, const dl_fcsm_options* options, const double* pose_in_submap_guess,
                       const float* high_resolution_points, int64_t n_high, const float* low_resolution_points,
                       int64_t n_low, const dl_grid* high_resolution_grid, const dl_grid* low_resolution_grid,
                       float min_score, dl_fcsm_result* result, float* all_scores, int64_t all_scores_capacity);

/* FastCorrelativeScanMatcher3D::Match (SM/fast_correlative_scan_matcher_3d.cc:145-162, :221-250, :296-350): the yaw search
 * around the node's orientation x the translation window. The yaw steps, the rotational scores (RotationalScanMatcher::Match on
 * the two histograms, rotational_scan_matcher.cc:123-155, :181-192) and the per-step poses are formed on the host exactly as the
 * reference does; every step that passes min_rotational_score becomes one translation search of the same device batch.
 * submap_histogram: the matcher's accumulated histogram (sum of the nodes' histograms rotated to the submap frame,
 * rotational_scan_matcher.cc:172-179); scan_histogram: the node's (TrajectoryNode::Data::rotational_scan_matcher_histogram);
 * gravity_alignment: quaternion w x y z. The fork's constraint builder calls dl_fcsm_match_3dof's form instead. */
int dl_fcsm_match(dl_context* ctx, const dl_fcsm_options* options, const float* submap_histogram, const float* scan_histogram,
                  int32_t histogram_size, const double* global_node_pose, const double* global_submap_pose,
                  const double* gravity_alignment, const float* high_resolution_points, int64_t n_high,
                  const float* low_resolution_points, int64_t n_low, const dl_grid* high_resolution_grid,
                  const dl_grid* low_resolution_grid, float min_score, dl_fcsm_result* result);

/* ---- scan_matching::CeresScanMatcher3D::Match (SM/ceres_scan_matcher_3d.h:41-61, .cc:63-123; options
 *      C/mapping/proto/scan_matching/ceres_scan_matcher_options_3d.proto + C/common/proto/ceres_solver_options.proto)
 * The Levenberg-Marquardt loop (Ceres 1.13 TrustRegionMinimizer semantics) runs entirely on the device. ------ */
#define DL_MAX_PAIRS 4
typedef struct dl_ceres_options {
  int32_t num_occupied_space_weights;
  double occupied_space_weight[DL_MAX_PAIRS];
  double translation_weight;
  double rotation_weight;
  int32_t only_optimize_yaw;
  int32_t use_nonmonotonic_steps;
  int32_t max_num_iterations;
  int32_t num_threads; /* accepted and ignored (ceres_solver_options.proto) */
} dl_ceres_options;
typedef struct dl_solve_summary { /* the subset of ceres::Solver::Summary the reference reads (LTB:543) + counters */
  double initial_cost;
  double final_cost;
  int32_t num_iterations; /* recorded iterations incl. iteration 0 */
  int32_t num_successful_steps;
  int32_t num_unsuccessful_steps;
  int32_t termination; /* 0 CONVERGENCE, 1 NO_CONVERGENCE, 2 FAILURE */
  int32_t num_evaluations;
  int32_t reserved;
} dl_solve_summary;
int dl_ceres_match(dl_context* ctx, const dl_ceres_options* options, const double* target_translation,
                   const double* initial_pose, int32_t num_pairs, const float* const* clouds, const int64_t* sizes,
                   const dl_grid* const* grids, double* pose_out, dl_solve_summary* summary);
/* `count` independent problems in one launch (the ConstraintBuilder3D fan-out, and multi-trajectory front ends).
 * Arrays are indexed [problem * num_pairs + pair]; poses / targets are count rows. */
int dl_ceres_match_batch(dl_context* ctx, const dl_ceres_options* options, int32_t count, int32_t num_pairs,
                         const double* target_translations, const double* initial_poses,
                         const float* const* clouds, const int64_t* sizes, const dl_grid* const* grids,
                         double* poses_out, dl_solve_summary* summaries);
/* Cost, local gradient (6) and J^T J (6x6 row-major) at `at_pose` — the quantities the device reduction feeds
 * to the LM loop — for kernel-level checks. */
int dl_ceres_normal_equations(dl_context* ctx, const dl_ceres_options* options, const double* target_translation,
                              const double* reference_pose, const double* at_pose, int32_t num_pairs,
                              const float* const* clouds, const int64_t* sizes, const dl_grid* const* grids,
                              double* cost, double* gradient6, double* hessian36);

/* ---- constraints::ConstraintBuilder3D::ComputeConstraint from the point where the pose guess is known
 *      (constraint_builder_3d.cc:261-333): coarse search (MatchWith3DofInitial, min_score prune) -> CeresScanMatcher3D::Match
 *      with the coarse pose as both initial pose and translation target -> Constraint{pose, weights, INTER_SUBMAP}.
 *      `count` independent (node, submap) pairs in one call, everything between the upload of the clouds and the download
 *      of the records stays on the device. Options = proto::ConstraintBuilderOptions (the fields this function reads).
 *      What stays on the host in the reference and here: SURF submap-to-submap matching and the frame bookkeeping that
 *      produce `pose_guesses` (:217-259), the sampler and the id maps. ----------------------------------------------- */
typedef struct dl_constraint_options {
  double min_score;
  double loop_closure_translation_weight;
  double loop_closure_rotation_weight;
  dl_fcsm_options fast_correlative_scan_matcher_3d;
  dl_ceres_options ceres_scan_matcher_3d; /* two occupied-space weights: high, low resolution */
} dl_constraint_options;
typedef struct dl_constraint { /* PoseGraphInterface::Constraint + the three scores ComputeConstraint histograms */
  int32_t found;               /* 0 <=> the reference leaves *constraint null */
  float score;
  float rotational_score;
  float low_resolution_score;
  double coarse_pose[7];       /* match_result->pose_estimate */
  double pose[7];              /* constraint_transform: submap i <- node j */
  double translation_weight;
  double rotation_weight;
  dl_solve_summary summary;
} dl_constraint;
/* Clouds are ragged: pair k uses points [offsets[k], offsets[k+1]) (xyz floats) of the high / low resolution arrays. */
int dl_constraint_search_batch(dl_context* ctx, const dl_constraint_options* options, int32_t count,
                               const double* pose_guesses, const float* high_resolution_points,
                               const int64_t* high_offsets, const float* low_resolution_points,
                               const int64_t* low_offsets, const dl_grid* const* high_resolution_grids,
                               const dl_grid* const* low_resolution_grids, dl_constraint* constraints);

/* ---- multi-GPU exchange steps (SURVEY 8e; BASELINE configs[3], [4]). One process per GPU. The reference farms the loop-closure
 *      searches out to a thread pool (constraint_builder_3d.cc:189-197) and hands every found constraint to the pose graph
 *      (:328-333); here the pairs are partitioned by SUBMAP OWNER (each grid resident on one GPU), every rank runs
 *      ConstraintBuilder3D::ComputeConstraint for its pairs on its device, and the constraint records are exchanged with ONE
 *      ncclAllGather over NVLink so that all ranks hold the same table. NCCL is loaded at run time (libnccl.so.2); the
 *      communicator is made from a 128-byte unique id the host program distributes (rank 0 calls dl_comm_unique_id). ----------- */
#define DL_COMM_ID_BYTES 128
typedef struct dl_comm dl_comm;
int dl_comm_unique_id(uint8_t* id128);
int dl_comm_create(dl_context* ctx, const uint8_t* id128, int32_t rank, int32_t world_size, dl_comm** out);
void dl_comm_destroy(dl_comm* comm);
int32_t dl_comm_rank(const dl_comm* comm);
int32_t dl_comm_world_size(const dl_comm* comm);
const char* dl_comm_last_error(void); /* errors of the calls that have no context (unique id) */
/* Thin device-buffer collectives on the communicator's context stream (asynchronous; dl_context_synchronize to wait). */
int dl_comm_all_gather_dev(dl_comm* comm, const void* send_dev, void* recv_dev, int64_t bytes_per_rank);
int dl_comm_all_reduce_f64_dev(dl_comm* comm, double* buffer_dev, int64_t count);
int dl_comm_broadcast_dev(dl_comm* comm, void* buffer_dev, int64_t bytes, int32_t root);

typedef struct dl_constraint_row { /* 96 bytes; PoseGraphInterface::Constraint as it crosses NVLink */
  int32_t submap_id, node_id;
  int32_t found;                  /* 1 found, 0 searched and pruned (the reference's null constraint), -1 padding */
  int32_t rank;                   /* who searched it */
  float score, low_resolution_score;
  double pose[7];                 /* constraint_transform: submap <- node */
  double translation_weight, rotation_weight;
} dl_constraint_row;
typedef struct dl_exchange_info {
  int64_t bytes_sent;             /* per rank: capacity * sizeof(dl_constraint_row) */
  int64_t bytes_received;         /* world_size * bytes_sent */
  float collective_ms;            /* device time of the ncclAllGather alone (CUDA events on the context's stream) */
  int32_t found_total;
} dl_exchange_info;
/* dl_constraint_search_batch for this rank's `count` pairs (count <= capacity; capacity is the same on every rank, e.g. the
 * largest shard), then the all-gather. table receives world_size * capacity rows, rank r's at [r * capacity, (r+1) * capacity),
 * unused slots with found = -1; identical on every rank. Between the upload of the clouds and the download of the table
 * everything stays on the device; the rows are packed by a kernel straight into the all-gather's send buffer. */
int dl_constraint_search_exchange(dl_context* ctx, dl_comm* comm, const dl_constraint_options* options, int32_t count,
                                  int32_t capacity, const int32_t* submap_ids, const int32_t* node_ids, const double* pose_guesses,
                                  const float* high_resolution_points, const int64_t* high_offsets,
                                  const float* low_resolution_points, const int64_t* low_offsets,
                                  const dl_grid* const* high_resolution_grids, const dl_grid* const* low_resolution_grids,
                                  dl_constraint_row* table, dl_exchange_info* info);

/* ---- optimization::OptimizationProblem3D::Solve as this fork runs it (C/mapping/internal/optimization/optimization_problem_3d.cc:259-589
 *      with the IMU / consecutive-node terms commented out there): sparse pose adjustment over the SpaCostFunction3D constraints
 *      (cost_functions/spa_cost_function_3d.h:35-58), first submap's translation constant and yaw fixed, LM as pose_graph.lua sets
 *      it. Block-sparse: every SpaCostFunction3D joins one submap and one node, so the node blocks are eliminated (Schur
 *      complement) and only the submaps' reduced system is factored densely, in one CTA.
 *      poses: num_submaps submap poses then num_nodes node poses, 7 doubles each (t xyz, q wxyz), in-out, identical on every
 *      rank. constraints: THIS RANK'S share (e.g. the rows it contributed to dl_constraint_search_exchange); with a communicator
 *      the per-rank blocks of the normal equations are summed by one ncclAllReduce(fp64) per evaluation and every rank returns
 *      the same poses. comm may be NULL (single process: all constraints local).
 *      frozen: num_submaps + num_nodes flags (NULL = none); a frozen pose is constant (OptimizationProblem3D::Solve's
 *      frozen_trajectories, optimization_problem_3d.cc:283-329): it has no parameters, and if it is the first submap its rotation
 *      is constant too. Constraints between two frozen poses only add a fixed cost: initial_cost / final_cost include it (as
 *      Ceres 1.13 reports them) while the tolerances see the rest. A pose that no constraint refers to (on any rank) is left out
 *      of the minimised program like a frozen one (Ceres removes unused parameter blocks): it comes back unchanged and does not
 *      enter ||x||, so it does not widen the parameter tolerance. The ranks learn which poses are referenced from the pair lists
 *      they exchange anyway (a pose that is not frozen and is referenced sits in a live constraint). With no parameters left the poses come back unchanged,
 *      termination CONVERGENCE, no iterations.
 *      Deterministic: no floating-point atomics; two calls on the same input return bit-identical poses, and with a communicator
 *      every rank does identical work after the all-reduce.
 *      Errors (DL_ERR_ARG, all detected before the first collective except the last, which every rank detects together after the
 *      set-up all-gather): an index outside the graph; more than DL_POSE_GRAPH_MAX_REDUCED parameters over the submaps that are
 *      not frozen (referenced or not: which submaps the constraints refer to is only known after the exchange); a graph whose
 *      submap / node counts, frozen poses, fix_z or iteration limit differ between the ranks. A device-memory
 *      reservation made after the first collective is agreed on by all ranks (a one-int all-gather), so every rank returns the
 *      same failure instead of one leaving its peers waiting. ------------------------------------------------------------- */
typedef struct dl_spa_constraint { /* PoseGraphInterface::Constraint: node j observed from submap i */
  int32_t submap, node;
  double zbar[7];
  double translation_weight, rotation_weight;
} dl_spa_constraint;
typedef struct dl_pose_graph_options {
  int32_t max_num_iterations; /* pose_graph.lua optimization_problem.ceres_solver_options.max_num_iterations (50) */
  int32_t fix_z;              /* optimization_problem.fix_z_in_3d */
} dl_pose_graph_options;
#define DL_POSE_GRAPH_MAX_REDUCED 3072
typedef struct dl_pose_graph_sparse_info {
  int32_t num_local_parameters;   /* live parameters of all poses (neither frozen nor unreferenced) */
  int32_t all_reduce_count;       /* one per evaluation */
  int64_t all_reduce_bytes;       /* per all-reduce: 8 * (2 + 42 * (num_submaps + num_nodes) + 36 * num_pairs) */
  float all_reduce_ms;            /* summed device time of the all-reduces (CUDA events) */
  float all_reduce_min_ms;        /* fastest single all-reduce */
  int32_t num_reduced_parameters; /* size of the factored system: the live parameters of the submaps (unreferenced ones have none) */
  int32_t num_pairs;              /* distinct (submap, node) pairs with a constraint not between two frozen poses, all ranks */
  int64_t setup_exchange_bytes;   /* received by this rank in the set-up all-gathers (0 without a communicator):
                                     world * (32 + 4), plus world * (4 + 8 * largest per-rank pair count) if any rank has pairs */
} dl_pose_graph_sparse_info;
int dl_pose_graph_solve_sparse(dl_context* ctx, dl_comm* comm, const dl_pose_graph_options* options, int32_t num_submaps,
                               int32_t num_nodes, double* poses, const uint8_t* frozen, const dl_spa_constraint* constraints,
                               int32_t num_constraints, dl_solve_summary* summary, dl_pose_graph_sparse_info* info);
/* The factors of dl_pose_graph_solve_sparse alone, at the given poses (same layout, frozen flags and fix_z; options'
 * max_num_iterations is not read): for each constraint its residual (6, into residuals[6 k ..]) and its Jacobian in the local
 * parameters (6 x 12 row-major into jacobians[72 k ..]: columns 0..5 the submap's, 6..11 the node's slots, the first dim of
 * each live and the rest zero; dim = 0 frozen, 2 the first submap (ConstantYawQuaternionPlus), else 3 + (fix_z ? 2 : 3)). */
int dl_pose_graph_evaluate(dl_context* ctx, const dl_pose_graph_options* options, int32_t num_submaps, int32_t num_nodes,
                           const double* poses, const uint8_t* frozen, const dl_spa_constraint* constraints, int32_t num_constraints,
                           double* residuals, double* jacobians);

/* ---- mapping::PoseGraph3D (C/mapping/internal/3d/pose_graph_3d.cc) on the fork's live loop-closure path: the object between the
 *      local trajectory builder and the optimizer. dl_pose_graph_3d_add_node restates, synchronously and in this order:
 *        1. AddNode (:112-144): the node's index; a new submap id when insertion_submaps.back() is new; the node's pose
 *           GetLocalToGlobalTransform * local_pose.
 *        2. the node's high- and low-resolution clouds are uploaded ONCE into the object's device node store; every later
 *           loop-closure search reads them there.
 *        3. ComputeConstraintsForNode (:335-399): InitializeGlobalSubmapPoses (:67-110, both branches), the node's global pose
 *           (:345-347), one INTRA_SUBMAP constraint local_submap^-1 * local_pose per insertion submap (matcher weights).
 *        4. if insertion_submaps.front() is finished (:138, :384-391): it is marked finished and `matches` (the output of the
 *           host SURF / RANSAC stage, ExtractFeaturesForSubmap, constraint_builder_3d.cc:436-532) are fanned out as
 *           ComputeConstraintsBetweenSubmaps does (:162-200): per matched submap, in (trajectory, index) order, the counter j
 *           restarts and runs over the finished submap's nodes in id order; a node with j % every_nodes_to_find_constraint != 0
 *           or already in computed_constraints_ for the target submap is skipped. The pose guess is (:226-259)
 *           T_G1_S1 * Embed3D(match) * T_S2_G2 * local_submap_from^-1 * local_pose with the rotation-only, yaw-removed gravity
 *           alignments of the two submaps' LOCAL poses (ComputeConstraintsForSubmap, :1075-1097, passes the local pose). All
 *           pairs of the submap run as one dl_constraint_search_batch (same kernels, same results) whose clouds are read from
 *           the node store. Found constraints enter computed_constraints_ and wait as pending.
 *        5. ++num_nodes_since_last_loop_closure; if optimize_every_n_nodes > 0 and the count is GREATER than it (:395-398), the
 *           optimization runs: the pending constraints are appended in search order, skipping a (submap, node) already in the
 *           table under either tag (HandleWorkQueue, :450-463); dl_pose_graph_solve_sparse over submaps then nodes, each ordered
 *           by (trajectory, index), with the frozen trajectories' poses frozen; RunOptimization's update (:734-764); the count
 *           is reset.
 *      dl_pose_graph_3d_run_final_optimization runs the same step. The fork sets max_num_final_iterations and then overwrites it
 *      with the regular cap (:677-682), so the final optimization uses optimization_problem.max_num_iterations as well.
 *      Rejected with DL_ERR_ARG, the graph unchanged: a match naming an unknown or unfinished submap, the finished submap itself,
 *      a same-trajectory submap with |index difference| <= 2 (ExtractFeaturesForSubmap never yields these, :466-473) or a
 *      submap twice; matches when no submap finished; insertion submaps that do not continue the trajectory's sequence (a new
 *      submap whose index is not the trajectory's next one). Graph state is committed only after the device work of steps 2-4
 *      succeeded. If the solve of step 5 fails, the node stays added, the poses stay those of the previous optimization and
 *      the found constraints stay pending (the next optimization appends them); the call returns the solve's status.
 *      Deliberate differences: execution is synchronous and deterministic (the reference's thread pool may or may not finish a
 *      search before WhenDone); not built: the per-node proximity search (its MaybeAdd*Constraint bodies are commented out in
 *      this fork, :205-323, :367-381), trajectory connectivity and global-localization sampling, landmark / fixed-frame /
 *      odometry / IMU terms, .pbstream loading, and a communicator (one GPU; the search and the solve it calls have NCCL
 *      variants).
 *      The submap grids are borrowed (owner: the caller, e.g. the dl_local_trajectory_builder) and must outlive the graph, or
 *      their submap's trim (see dl_pg3d_last_trimmed).
 *
 *      Pure localization (MapBuilder with pure_localization, map_builder.cc:147-151): the dl_pg3d_* calls below. Their prefix is
 *      the block's type prefix; the dl_pose_graph_3d_* entry points above are the mapping path.
 *      Ids with holes: submaps and nodes are MapById per trajectory (C/mapping/id.h). A trim removes one id; trimming a
 *      trajectory's highest submap (node) index forbids appending submaps (nodes) to it (id.h:289-300), and an add_node that
 *      would append one returns DL_ERR_ARG, the graph unchanged. The solve's submap and node order, the fan-out over a
 *      finished submap's node ids and GetLocalToGlobalTransform's last optimized submap skip the holes; the solve holds its
 *      first remaining submap (OptimizationProblem3D::Solve's first_submap, optimization_problem_3d.cc:286-316). A match or
 *      an insertion submap naming a trimmed submap is rejected like an unknown one.
 *      Trimmers (HandleWorkQueue, :492-501) run at the end of every successful optimization (the periodic one of add_node,
 *      dl_pose_graph_3d_run_final_optimization, dl_pg3d_finish_trajectory) in the order they were added; a finished trimmer
 *      is dropped; a failed solve runs none. Trimmed nodes' clouds become dead ranges of the node store; when the dead floats
 *      exceed the live ones and number at least 2^20 (4 MiB), kernel pg3d_store_compact copies every live node's clouds into
 *      a fresh store in one launch and the old one is freed, so after every trim used <= 2 * live or used - live < 4 MiB
 *      (dl_pg3d_store_usage), and the copying costs O(1) per uploaded float. A failed compaction leaves the old store and
 *      offsets as they were and returns DL_ERR_CUDA; the trim itself stands. A graph on which no dl_pg3d_* call is made
 *      behaves exactly as without them. ---- */
typedef struct dl_pose_graph_3d dl_pose_graph_3d;
typedef struct dl_pose_graph_3d_options { /* proto::PoseGraphOptions, the fields this path reads */
  int32_t optimize_every_n_nodes;         /* 0: only on dl_pose_graph_3d_run_final_optimization */
  int32_t every_nodes_to_find_constraint; /* constraint_builder.every_nodes_to_find_constraint (>= 1) */
  double matcher_translation_weight;      /* INTRA_SUBMAP weights */
  double matcher_rotation_weight;
  dl_constraint_options constraint_builder;
  dl_pose_graph_options optimization_problem;
} dl_pose_graph_3d_options;
typedef struct dl_pg3d_insertion_submap {  /* one of InsertionResult::insertion_submaps */
  int32_t submap_index;                    /* index in its trajectory (dl_matching_result::insertion_submap_index) */
  int32_t finished;                        /* Submap3D::finished() after the node's insertion */
  const dl_grid* high_resolution_grid;     /* borrowed */
  const dl_grid* low_resolution_grid;
  double local_pose[7];
} dl_pg3d_insertion_submap;
typedef struct dl_pg3d_node {              /* TrajectoryNode::Data + the insertion submaps */
  int32_t trajectory_id;
  int32_t num_insertion_submaps;           /* 1 or 2 */
  double time;
  double local_pose[7];
  const float* high_resolution_points;     /* xyz floats, tracking frame */
  int64_t num_high_resolution;
  const float* low_resolution_points;
  int64_t num_low_resolution;
  dl_pg3d_insertion_submap insertion_submaps[2];
} dl_pg3d_node;
typedef struct dl_pg3d_submap_match {      /* one entry of matched_submaps: an earlier finished submap + Rigid2d (x, y, theta) */
  int32_t trajectory_id;
  int32_t submap_index;
  double x, y, theta;
} dl_pg3d_submap_match;
typedef struct dl_pg3d_add_node_info {
  int32_t node_index;                      /* NodeId::node_index in its trajectory */
  int32_t num_searched;                    /* (node, submap) pairs searched by this call */
  int32_t num_found;                       /* ... of which the coarse search passed min_score */
  int32_t optimized;                       /* 1 if this call ran the optimization */
  int64_t cloud_bytes_uploaded;            /* host-to-device bytes of point clouds: 12 * (n_hi + n_lo) of this node, nothing else */
  double bookkeeping_ms, search_ms, solve_ms; /* host wall time of the call's parts (each ends in a device synchronise) */
  dl_solve_summary summary;                /* of the optimization, if optimized */
} dl_pg3d_add_node_info;
#define DL_PG3D_INTRA_SUBMAP 0
#define DL_PG3D_INTER_SUBMAP 1
typedef struct dl_pg3d_constraint {        /* PoseGraphInterface::Constraint */
  int32_t submap_trajectory_id, submap_index;
  int32_t node_trajectory_id, node_index;
  double zbar[7];
  double translation_weight, rotation_weight;
  int32_t tag;                             /* DL_PG3D_INTRA_SUBMAP / DL_PG3D_INTER_SUBMAP */
  int32_t reserved;
} dl_pg3d_constraint;
int dl_pose_graph_3d_create(dl_context* ctx, const dl_pose_graph_3d_options* options, dl_pose_graph_3d** out);
void dl_pose_graph_3d_destroy(dl_pose_graph_3d* graph);
/* matches: num_matches entries, only when insertion_submaps[0].finished (else num_matches must be 0). info may be NULL. */
int dl_pose_graph_3d_add_node(dl_pose_graph_3d* graph, const dl_pg3d_node* node, int32_t num_matches,
                              const dl_pg3d_submap_match* matches, dl_pg3d_add_node_info* info);
int dl_pose_graph_3d_freeze_trajectory(dl_pose_graph_3d* graph, int32_t trajectory_id);
/* summary may be NULL. With no submap in the graph it returns DL_OK and leaves summary zeroed. */
int dl_pose_graph_3d_run_final_optimization(dl_pose_graph_3d* graph, dl_solve_summary* summary);
/* Poses of one trajectory, 7 doubles each, in index order. which:
 *   DL_PG3D_NODE_POSES          trajectory_nodes_' global poses (GetTrajectoryNodePoses);
 *   DL_PG3D_SUBMAP_POSES        GetSubmapDataUnderLock (:937-952): the optimized pose, or local_to_global * local_pose for a
 *                               submap not optimized yet;
 *   DL_PG3D_OPTIMIZATION_NODES  / DL_PG3D_OPTIMIZATION_SUBMAPS  the optimization problem's node_data / submap_data, i.e. the
 *                               poses the next solve starts from.
 * Pass poses = NULL to query *count (the trajectory's size; 0 for an unknown trajectory). */
#define DL_PG3D_NODE_POSES 0
#define DL_PG3D_SUBMAP_POSES 1
#define DL_PG3D_OPTIMIZATION_NODES 2
#define DL_PG3D_OPTIMIZATION_SUBMAPS 3
int dl_pose_graph_3d_poses(const dl_pose_graph_3d* graph, int32_t trajectory_id, int32_t which, int32_t capacity, double* poses,
                           int32_t* count);
/* GetLocalToGlobalTransform (:914-935): last optimized submap's global pose * its local pose^-1 (identity before any). */
int dl_pose_graph_3d_local_to_global(const dl_pose_graph_3d* graph, int32_t trajectory_id, double* pose);
/* The constraint table in insertion order. Pass out = NULL to query *count. */
int dl_pose_graph_3d_constraints(const dl_pose_graph_3d* graph, int32_t capacity, dl_pg3d_constraint* out, int32_t* count);
/* The (node, submap) searches of the last successful dl_pose_graph_3d_add_node call in search order: ids, the pose guess and the
 * dl_constraint_search_batch record. Pass out = NULL to query *count. */
typedef struct dl_pg3d_search {
  int32_t submap_trajectory_id, submap_index;
  int32_t node_trajectory_id, node_index;
  double pose_guess[7];
  dl_constraint result;
} dl_pg3d_search;
int dl_pose_graph_3d_last_searches(const dl_pose_graph_3d* graph, int32_t capacity, dl_pg3d_search* out, int32_t* count);
/* Bytes of clouds uploaded into the node store since creation, and its capacity in bytes. */
int dl_pose_graph_3d_store_bytes(const dl_pose_graph_3d* graph, int64_t* uploaded, int64_t* capacity);
typedef struct dl_pg3d_submap_id {         /* SubmapId */
  int32_t trajectory_id, submap_index;
} dl_pg3d_submap_id;
/* TrimmingHandle::MarkSubmapAsTrimmed (:1002-1058): nodes_to_retain = the nodes with an INTRA_SUBMAP constraint to another
 * submap; every constraint of the submap is dropped; the nodes left without an INTRA_SUBMAP constraint and every constraint
 * of theirs are dropped; the submap and those nodes leave the graph and the optimization problem (optimization_problem_3d.cc:
 * 229-251). DL_ERR_ARG, the graph unchanged: an unknown or already trimmed submap, an unfinished submap (the reference
 * CHECKs), or constraints still pending (there are none right after an optimization, which is where trimmers run). */
int dl_pg3d_trim_submap(dl_pose_graph_3d* graph, int32_t trajectory_id, int32_t submap_index);
/* PureLocalizationTrimmer (C/mapping/pose_graph_trimmer.cc:24-45): after each optimization, every submap of the trajectory but
 * the newest num_submaps_to_keep (in index order) is trimmed; once the trajectory is finished all of them are, and the trimmer
 * is done. num_submaps_to_keep < 3: DL_ERR_ARG. */
int dl_pg3d_add_pure_localization_trimmer(dl_pose_graph_3d* graph, int32_t trajectory_id, int32_t num_submaps_to_keep);
/* FinishTrajectory (:535-547): every submap of the trajectory becomes finished, then the step of
 * dl_pose_graph_3d_run_final_optimization runs (pending constraints appended, solve, update, trimmers). The trajectory stays
 * finished if that solve fails. Finishing twice returns DL_ERR_ARG; so does dl_pose_graph_3d_add_node on a finished
 * trajectory. */
int dl_pg3d_finish_trajectory(dl_pose_graph_3d* graph, int32_t trajectory_id);
int dl_pg3d_is_trajectory_finished(const dl_pose_graph_3d* graph, int32_t trajectory_id, int32_t* finished);
/* SetInitialTrajectoryPose (:849-856) with GetInterpolatedGlobalTrajectoryPose (:858-876, used at :914-928): while trajectory
 * `from` has no optimized submap, its local-to-global transform is the `to` trajectory's node global poses interpolated at
 * `time`, times relative_pose (t xyz, q wxyz). The interpolation takes the first node whose time is not below `time`
 * (lower_bound); before the first node it is the first node's pose, past the last the last one's; else
 * transform::Interpolate of the node before it and it: factor = (time - t0) / (t1 - t0) from the dl_pg3d_node::time doubles,
 * translation t0 + (t1 - t0) * factor, rotation Eigen's slerp. `to` without nodes when the transform is needed: the call
 * that needs it (add_node of `from`, the poses or local_to_global query) returns DL_ERR_ARG (the reference CHECKs). */
int dl_pg3d_set_initial_trajectory_pose(dl_pose_graph_3d* graph, int32_t from_trajectory_id, int32_t to_trajectory_id,
                                        const double* relative_pose, double time);
/* The indices of the rows dl_pose_graph_3d_poses returns for the same `which` (submaps or nodes still in the graph, in index
 * order). Pass indices = NULL to query *count. */
int dl_pg3d_ids(const dl_pose_graph_3d* graph, int32_t trajectory_id, int32_t which, int32_t capacity, int32_t* indices,
                int32_t* count);
/* The submaps trimmed by the last dl_pose_graph_3d_add_node, dl_pose_graph_3d_run_final_optimization, dl_pg3d_finish_trajectory
 * or dl_pg3d_trim_submap call, in trim order; each of these calls empties the list when it starts, so after a call that failed
 * (a rejection, or a failure after some trims had already been made) it holds exactly what that call trimmed. Their grids are
 * no longer read by the graph: the caller may release them (dl_ltb_release_submap). Pass out = NULL to query *count. */
int dl_pg3d_last_trimmed(const dl_pose_graph_3d* graph, int32_t capacity, dl_pg3d_submap_id* out, int32_t* count);
/* The node store in bytes: live (the clouds of the nodes still in the graph), used (written, dead ranges included), capacity. */
int dl_pg3d_store_usage(const dl_pose_graph_3d* graph, int64_t* live_bytes, int64_t* used_bytes, int64_t* capacity_bytes);

/* ---- IMU: pre-integration (LocalTrajectoryBuilder3D::AddImuData, LTB:164-201, with the in-repo mid-point integrator
 *      C/mapping/internal/3d/initialization/integration_base.h:109-265 instead of the un-vendored GTSAM one) and the
 *      scan match with the pre-integration residual (integration_base.h:267-301) fused into the same solve.
 *      The fused solve is an EXTENSION asked for by BASELINE.json: the reference chains CeresScanMatcher3D::Match and a
 *      GTSAM iSAM2 update (LTB:535-555, :693-863). State order everywhere: p, theta, v, b_a, b_g. ------------------- */
typedef struct dl_imu_noise { /* C/mapping/proto/imu_options.proto: acc_noise, gyr_noise, acc/gyr bias random walk */
  double acc_n, gyr_n, acc_w, gyr_w;
} dl_imu_noise;
typedef struct dl_preintegration {
  double sum_dt;
  double delta_p[3], delta_q[4], delta_v[3];  /* delta_q is w x y z */
  double linearized_ba[3], linearized_bg[3];
  double jacobian[225], covariance[225];       /* row-major 15 x 15 */
} dl_preintegration;
typedef struct dl_nav_state { /* X(k), V(k), B(k) of the reference's window (LTB:708-852) */
  double p[3], q[4], v[3], ba[3], bg[3];
} dl_nav_state;
/* `count` intervals; interval k uses samples [offsets[k], offsets[k+1]) of dt / acc (xyz) / gyr (xyz); the first
 * sample of an interval only latches the integrator (integration_base.h:111-118). biases: 6 doubles per interval. */
int dl_imu_preintegrate(dl_context* ctx, const dl_imu_noise* noise, int32_t count, const int32_t* offsets,
                        const double* dt, const double* acc, const double* gyr, const double* biases,
                        dl_preintegration* out);
/* State at the end of the interval (the front end's pose prediction, LTB:188-199). gravity: 3 doubles (+9.8 z). */
int dl_imu_predict(const dl_nav_state* state_i, const dl_preintegration* m, const double* gravity, dl_nav_state* state_j);
/* The IMU factor of the fused solve alone, for kernel-level checks: the device preparation of dl_frontend_match_batch_imu_samples
 * (prediction, factor in the submap frame, information matrix) followed by the solve's IMU normal equations, for `count`
 * independent (states_i[k], preintegrations[k], submap_local_poses[k]) triples. x16: 16 doubles per factor (p q v ba bg of
 * state j in the SUBMAP frame) at which the equations are evaluated, or NULL for the prepared start (the prediction).
 * Outputs per factor: ok (0: the covariance is not positive definite, every other output of the factor is zero), the
 * predicted state (local frame), information = imu_weight^2 * covariance^-1 (225, row-major), residual (15), hessian = J^T W J
 * (225), gradient = J^T W r (15) and cost2 = r^T W r. Order p, theta, v, b_a, b_g; theta perturbs q on the left
 * (q <- (cos|d|, sin|d|/|d| d) (x) q). */
int dl_imu_factor_evaluate(dl_context* ctx, int32_t count, const dl_nav_state* states_i, const dl_preintegration* preintegrations,
                           const double* submap_local_poses, const double* gravity, double imu_weight, const double* x16,
                           int32_t* ok, dl_nav_state* predicted, double* information, double* residual, double* hessian,
                           double* gradient, double* cost2);
/* Fused scan match for `count` independent problems: state i fixed, the 15 local parameters of state j estimated
 * from the occupied-space residuals (+ optional translation / rotation priors of `options`) and the IMU residual
 * weighted by imu_weight^2 * covariance^-1. States are in the local frame; submap_local_poses (7 doubles each) place
 * the grids. Arrays indexed like dl_ceres_match_batch. preintegrations[k] may be linearised at other biases than
 * states_i[k]'s: the factor then takes the first-order bias correction of integration_base.h:283-290 (delta_p, delta_v
 * and delta_q moved by the bias blocks of the pre-integration's Jacobian), as the window smoother does. */
int dl_fused_match_batch(dl_context* ctx, const dl_ceres_options* options, double imu_weight, const double* gravity,
                         int32_t count, int32_t num_pairs, const double* submap_local_poses,
                         const dl_nav_state* states_i, const dl_nav_state* initial_states_j,
                         const dl_preintegration* preintegrations, const float* const* clouds, const int64_t* sizes,
                         const dl_grid* const* grids, dl_nav_state* states_j_out, dl_solve_summary* summaries);

/* ---- the reference's TWO-STAGE mode, second stage: LocalTrajectoryBuilder3D::WindowOptimize (LTB:693-863) as a fixed-lag smoother
 *      on the device, no GTSAM. Per trajectory: the previous key x_i with its carried marginal (prior), the IMU factor between x_i
 *      and the new key x_j (the in-repo pre-integration residual with first-order bias correction, integration_base.h:267-301,
 *      weighted by its propagated covariance; the last six rows are the bias random walk), the scan matcher's pose as a prior on
 *      x_j with diagonal sigmas (ceres_pose_noise_{t,r}, LTB:94-101, :815-818), optionally the gravity-direction prior
 *      (gravity_factor.cc:10-31). Gauss-Newton on the 30 local parameters, then the Schur complement on x_i: the information of
 *      x_j, which is the next call's prior — what iSAM2's marginal of the newest key carries between the reference's re-seeds
 *      (LTB:750-797). Tangent order everywhere: p, theta, v, b_a, b_g; rotations perturb on the left, q <- exp(theta) q with
 *      |theta| the HALF angle (the chart of dl_fused_match_batch). GTSAM's own integrator / factor are not restated (neither
 *      library is in this image): parity of this row is oracle <-> device. ------------------------------------------------ */
typedef struct dl_window_options {
  double pose_sigma_translation; /* imu_options.ceres_pose_noise_t */
  double pose_sigma_rotation;    /* imu_options.ceres_pose_noise_r (on 2 vec(q_m^-1 q_j), i.e. the full angle) */
  double imu_weight;             /* scales the IMU factor's square-root information (1 = the propagated covariance as is) */
  double gravity[3];             /* +9.8 z: the convention of integration_base.h:292-297 */
  int32_t max_num_iterations;    /* Gauss-Newton iterations (10 when 0) */
  int32_t use_gravity_factor;
  double gravity_sigma;          /* imu_options.prior_gravity_noise */
  double gravity_direction[3];   /* estimated up direction in the local frame (g_vec_est_G_) */
  double body_reference_direction[3]; /* the reference direction in the body frame that should map to it */
} dl_window_options;
/* gravity_direction and body_reference_direction are directions: with use_gravity_factor set, a zero or non-finite one is
 * DL_ERR_ARG and both are normalised before use (as gtsam::Unit3 does), so their lengths do not change the result. The factor
 * differs from gravity_factor.cc in two stated ways: b_ref is rotated by the whole R_j, not by its roll and pitch only
 * (Rot3::RzRyRx(r.x, r.y, 0)), and the residual carries no k_cost_value = 1e-5 offset. */
/* `count` independent trajectories. prior_information: 225 doubles each (row-major 15 x 15). matched_poses: 7 each.
 * initial_states_j may be NULL (start from the IMU prediction). states_i_out (optional) receives the smoothed previous keys.
 * summaries[k].termination: 0 converged, 1 iteration limit, 2 a covariance / system was not positive definite (no output). */
int dl_window_optimize_batch(dl_context* ctx, const dl_window_options* options, int32_t count, const dl_nav_state* states_i,
                             const double* prior_information, const dl_preintegration* preintegrations, const double* matched_poses,
                             const dl_nav_state* initial_states_j, dl_nav_state* states_i_out, dl_nav_state* states_j_out,
                             double* information_out, dl_solve_summary* summaries);
/* The window's factors alone, for kernel-level checks: for `count` problems (arguments as dl_window_optimize_batch) evaluated at
 * the given (x_i[k], x_j[k]) — x_i need not be the prior mean states_i[k]. Outputs per problem: ok (0: the IMU covariance is not
 * positive definite, every other output of the problem is zero), residuals (38: 15 prior, 15 IMU, 6 pose, 2 gravity; the gravity
 * rows are 0 without the factor), jacobians (38 x 30 row-major, d r / d (delta_i, delta_j) in the tangent order and chart above)
 * and weights (38 x 38 row-major, block diagonal: prior information, imu_weight^2 covariance^-1, 1 / sigma^2 of the pose and
 * gravity rows). The solve minimises 1/2 r^T W r. */
int dl_window_evaluate(dl_context* ctx, const dl_window_options* options, int32_t count, const dl_nav_state* states_i,
                       const double* prior_information, const dl_preintegration* preintegrations, const double* matched_poses,
                       const dl_nav_state* x_i, const dl_nav_state* x_j, int32_t* ok, double* residuals, double* jacobians,
                       double* weights);

/* ---- the per-scan front end of LocalTrajectoryBuilder3D::AddRangeData / AddAccumulatedRangeData
 *      (LTB:393-554): voxel filter -> deskew/transform/range gate -> voxel filter -> adaptive filters ->
 *      [RT-CSM] -> Ceres match, for a batch of independent scans against one submap. ---------------------------- */
typedef struct dl_frontend_options { /* C/mapping/proto/3d/local_trajectory_builder_options_3d.proto */
  float min_range;
  float max_range;
  float voxel_filter_size;
  dl_adaptive_voxel_filter_options high_resolution_adaptive_voxel_filter;
  dl_adaptive_voxel_filter_options low_resolution_adaptive_voxel_filter;
  int32_t use_online_correlative_scan_matching;
  /* layout of the `ranges` rows: 8 (default when 0) = RangeMeasurement {x y z t, u64 origin index} as produced by
   * RangeDataSynchronizer; 4 = sensor::TimedPointCloud rows {x y z t} of a single sensor (origin index 0), the
   * layout AddRangeData itself receives (timed_point_cloud_data.h:27-31) — half the host-to-device bytes; 3 = bare x y z
   * rows with the times given as runs (time_run_* below) — three eighths. */
  int32_t range_row_floats;
  double scan_period;
  dl_rtcsm_options real_time_correlative_scan_matcher;
  dl_ceres_options ceres_scan_matcher;
  /* Host-buffer calls only. 0: ranges[b] are unrelated buffers, one upload per scan. > 0: the caller guarantees that the
   * scans sit in ONE allocation at a constant stride, ranges[b] == (char*)ranges[0] + b * stride * row bytes with
   * stride >= every sizes[b]; each sub-batch is then uploaded by a single strided copy (rows between a scan's end and the
   * next scan's start are read but ignored). Checked against the pointers; DL_ERR_ARG if they disagree. */
  int64_t host_scan_stride_rows;
  /* range_row_floats == 3 only: rows are bare {x y z} (12 bytes) and the per-point times come as RUNS — a spinning LiDAR stamps a
   * whole firing column with one time, so a 130k-point sweep has ~2k distinct times. Scan k owns runs
   * [time_run_offsets[k], time_run_offsets[k+1]); run r starts at row time_run_first_row[r] of its scan (ascending, the first is 0)
   * and all rows up to the next run's first row carry time_run_value[r]. The deskew sees exactly the floats the 16-byte rows
   * would carry (bit-identical results) while the host-to-device copy shrinks by a quarter. Single sensor (origin index 0). */
  const int32_t* time_run_offsets;
  const int32_t* time_run_first_row;
  const float* time_run_value;
} dl_frontend_options;

typedef struct dl_scan_result {
  double pose_estimate_local[7];          /* matching_submap->local_pose() * pose_observation_in_submap (LTB:553) */
  double pose_observation_in_submap[7];
  dl_solve_summary summary;
  float rtcsm_score;
  int32_t ok;                             /* 0 = dropped (empty cloud), like the reference's nullptr; -1 = a point lay
                                             outside the voxel-key span of the fused front half: +-2^(b-1) voxels of
                                             voxel_filter_size around the scan's pose, b = min(21, (63 - ceil(log2(capacity)))
                                             / 3), i.e. +-2.4 km at 0.15 m for scans up to 256 k points (results invalid;
                                             dl_voxel_filter itself has no limit); -2 = no IMU
                                             factor could be formed for this scan (dl_frontend_*_imu_samples) */
  int32_t num_first_filter, num_returns, num_misses, num_high_resolution, num_low_resolution;
  /* adaptive filter bookkeeping: points inside max_range and voxel passes run, per filter (high, low) */
  int32_t num_cropped_high, num_cropped_low, num_passes_high, num_passes_low;
  int32_t reserved;
} dl_scan_result;

/* ---- wire format -> TimedPointCloud rows (SensorBridge::HandlePointCloud2Message + HandleRangefinder,
 *      cartographer_ros/sensor_bridge.cc:176-240, :286-300): decodes the points of a sensor_msgs/PointCloud2 message
 *      (`num_points` records of `point_step` bytes; x / y / z float32 at their field offsets), drops NaN / Inf points,
 *      makes the per-point time relative to the LAST point of the message and moves the points into the tracking frame.
 *      time_type follows the reference's sensor types: FLOAT32_SECONDS = "velodyne" (field `time`), UINT32_NANOSECONDS =
 *      "ouster" (field `t`), FLOAT64_SECONDS = "robosense" (field `timestamp`), NONE = anything else (t = 0).
 *      Output rows are {x, y, z, t} floats = the 16-byte layout dl_frontend_* take with range_row_floats = 4.
 *      *stamp_offset_seconds is what the reference adds to the message stamp (velodyne / ouster: time of the last point). */
#define DL_TIME_NONE 0
#define DL_TIME_FLOAT32_SECONDS 1
#define DL_TIME_UINT32_NANOSECONDS 2
#define DL_TIME_FLOAT64_SECONDS 3
typedef struct dl_point_cloud2_layout {
  int32_t point_step;
  int32_t offset_x, offset_y, offset_z, offset_time;
  int32_t time_type;
} dl_point_cloud2_layout;
/* Host message in, host rows out (capacity num_points rows). */
int dl_decode_point_cloud2(dl_context* ctx, const dl_point_cloud2_layout* layout, const void* data, int64_t num_points,
                           const double* sensor_to_tracking, float* rows_out, int64_t* num_rows_out,
                           double* stamp_offset_seconds);
/* Device message in (e.g. uploaded as it arrived), device rows out: rows_out_dev has capacity num_points rows and can be
 * a slice of the buffer dl_frontend_match_batch_dev reads. The row count and stamp offset come back to the host. */
int dl_decode_point_cloud2_dev(dl_context* ctx, const dl_point_cloud2_layout* layout, const void* data_dev,
                               int64_t num_points, const double* sensor_to_tracking, float* rows_out_dev,
                               int64_t* num_rows_out, double* stamp_offset_seconds);

/* Scan ingest only (LTB:393-487): the batched front half of dl_frontend_match_batch run on one scan.
 * ranges: n RangeMeasurement rows (32 bytes: x y z t + uint64 origin index); origins: 3 floats per sensor.
 * Outputs have capacity n rows. counts_out[4] = {first filter survivors, returns (local frame, before 2nd filter),
 * returns in tracking frame, misses in tracking frame}. DL_ERR_ARG if a point lies outside the voxel-key span of
 * the second voxel filter (where a batched call would report ok = -1 for the scan, see dl_scan_result). */
int dl_ingest_scan(dl_context* ctx, const dl_frontend_options* options, const void* ranges, int64_t n,
                   const float* origins, int32_t num_origins, const double* prev_pose, const double* predicted_pose,
                   int64_t* first_keep_out, float* returns_local_out, float* returns_tracking_out,
                   float* misses_tracking_out, float* current_pose7f_out, int64_t* counts_out);

/* Whole hot path for `num_scans` scans; host buffers, copies included (this is the "e2e" call). */
int dl_frontend_match_batch(dl_context* ctx, const dl_frontend_options* options, int32_t num_scans,
                            const void* const* ranges, const int64_t* sizes, const float* origins,
                            int32_t num_origins, const double* prev_poses, const double* predicted_poses,
                            const double* submap_local_pose, const dl_grid* high_resolution_grid,
                            const dl_grid* low_resolution_grid, dl_scan_result* results);

/* dl_frontend_match_batch with the IMU pre-integration residual fused into every scan's solve (dl_fused_match_batch's
 * 15-parameter problem behind the same ingest / filter front half): scan k starts from state states_i[k] at the previous
 * scan, predicted_states[k] = dl_imu_predict(states_i[k], preintegrations[k]) provides the pose prediction (its pose is what
 * the plain call takes as predicted_poses; prev_poses[k] is states_i[k]'s pose) and the initial velocity and biases.
 * states_out[k] receives the estimated state of scan k (local frame); results[k] as in the plain call, with the pose part
 * of the state. preintegrations[k] may be linearised at other biases than states_i[k]'s (bias correction as in
 * dl_fused_match_batch). An EXTENSION like dl_fused_match_batch: the reference chains the plain match and a GTSAM update.
 * With use_online_correlative_scan_matching the correlative pre-match runs first (LTB:514-521) and its pose replaces the
 * pose part of state j's initial value; velocity and biases stay the prediction's, and the translation target of the
 * solve stays the prediction's translation (LTB:536). Combining the pre-match with the fused solve is part of the same
 * extension. This and every fused entry below refuse only_optimize_yaw (DL_ERR_ARG). */
typedef struct dl_frontend_imu {
  double imu_weight;
  double gravity[3];
  const dl_nav_state* states_i;
  const dl_nav_state* predicted_states;
  const dl_preintegration* preintegrations;
  dl_nav_state* states_out;
} dl_frontend_imu;
int dl_frontend_match_batch_imu(dl_context* ctx, const dl_frontend_options* options, const dl_frontend_imu* imu,
                                int32_t num_scans, const void* const* ranges, const int64_t* sizes, const float* origins,
                                int32_t num_origins, const double* submap_local_pose, const dl_grid* high_resolution_grid,
                                const dl_grid* low_resolution_grid, dl_scan_result* results);

/* The same front end fed with the RAW IMU samples between consecutive scans (configs[1]: 64-beam + 200 Hz IMU): the
 * pre-integration (LocalTrajectoryBuilder3D::AddImuData, LTB:164-201, integration_base.h:109-265), the state prediction that
 * seeds the pose and the deskew (LTB:188-199, :426-428), the factor's information matrix and the fused solve all run on the
 * device — nothing IMU-related is computed on the host. Scan k uses samples [offsets[k], offsets[k+1]) of dt / acc (xyz) /
 * gyr (xyz); the first sample of an interval only latches the integrator; states_i[k] is the optimised state at the previous
 * scan (its biases are the linearisation point). Result ok = -2 marks a scan whose interval has no usable samples
 * (covariance not positive definite): no solve ran for it. An EXTENSION like dl_fused_match_batch. */
typedef struct dl_frontend_imu_samples {
  dl_imu_noise noise;
  double imu_weight;
  double gravity[3];
  const dl_nav_state* states_i;
  const int32_t* offsets; /* num_scans + 1, offsets[0] == 0 */
  const double* dt;
  const double* acc;
  const double* gyr;
} dl_frontend_imu_samples;
/* Host scans in, results + estimated states (+ optionally the predicted states) out; blocking. */
int dl_frontend_match_batch_imu_samples(dl_context* ctx, const dl_frontend_options* options, const dl_frontend_imu_samples* imu,
                                        int32_t num_scans, const void* const* ranges, const int64_t* sizes, const float* origins,
                                        int32_t num_origins, const double* submap_local_pose, const dl_grid* high_resolution_grid,
                                        const dl_grid* low_resolution_grid, dl_scan_result* results, dl_nav_state* states_out,
                                        dl_nav_state* predicted_states_out);
/* Device-resident scans (layout as dl_frontend_match_batch_dev); results and states stay on the device. Only the IMU samples
 * and states_i (about 1.3 kB per scan) are uploaded. */
int dl_frontend_match_batch_imu_samples_dev(dl_context* ctx, const dl_frontend_options* options,
                                            const dl_frontend_imu_samples* imu, int32_t num_scans, const void* ranges_dev,
                                            int64_t cap_rows, const int64_t* sizes, const float* origins, int32_t num_origins,
                                            const double* submap_local_pose, const dl_grid* high_resolution_grid,
                                            const dl_grid* low_resolution_grid, dl_scan_result* results_dev,
                                            dl_nav_state* states_out_dev);
/* Streaming form (see dl_frontend_submit): the sample arrays must stay valid until the collect. */
int dl_frontend_submit_imu_samples(dl_context* ctx, const dl_frontend_options* options, const dl_frontend_imu_samples* imu,
                                   int32_t num_scans, const void* const* ranges, const int64_t* sizes, const float* origins,
                                   int32_t num_origins, const double* submap_local_pose, const dl_grid* high_resolution_grid,
                                   const dl_grid* low_resolution_grid);
int dl_frontend_collect_imu(dl_context* ctx, int32_t num_scans, dl_scan_result* results, dl_nav_state* states_out);

/* Streaming form of dl_frontend_match_batch: submit enqueues the uploads, every kernel and the download of the results into
 * pinned staging and returns WITHOUT waiting; collect blocks until that batch is finished and copies the results out.
 * One batch may be in flight per context; a caller that wants the upload of batch i+1 to overlap the tail of batch i
 * alternates between two contexts (grids are shared read-only between contexts of the same device), which is how
 * bench.py's e2e loop keeps the PCIe link busy. The host buffers must stay valid (and should be pinned) until collect.
 * Any other call on a context with a batch in flight fails with DL_ERR_ARG. */
int dl_frontend_submit(dl_context* ctx, const dl_frontend_options* options, int32_t num_scans, const void* const* ranges,
                       const int64_t* sizes, const float* origins, int32_t num_origins, const double* prev_poses,
                       const double* predicted_poses, const double* submap_local_pose,
                       const dl_grid* high_resolution_grid, const dl_grid* low_resolution_grid);
int dl_frontend_collect(dl_context* ctx, int32_t num_scans, dl_scan_result* results);

/* Device-resident variant: ranges_dev is ONE device buffer of num_scans * cap_rows RangeMeasurement rows; scan s
 * occupies rows [s * cap_rows, s * cap_rows + sizes[s]). Results stay in results_dev (device) until
 * dl_frontend_fetch_results copies them out. No scan data is copied from or to the host inside this call. */
int dl_frontend_match_batch_dev(dl_context* ctx, const dl_frontend_options* options, int32_t num_scans,
                                const void* ranges_dev, int64_t cap_rows, const int64_t* sizes,
                                const float* origins, int32_t num_origins, const double* prev_poses,
                                const double* predicted_poses, const double* submap_local_pose,
                                const dl_grid* high_resolution_grid, const dl_grid* low_resolution_grid,
                                dl_scan_result* results_dev);
int dl_frontend_fetch_results(dl_context* ctx, const dl_scan_result* results_dev, int32_t num_scans,
                              dl_scan_result* results);

/* ---- scan_matching::RotationalScanMatcher::ComputeHistogram (SM/rotational_scan_matcher.cc:31-121, :159-170) on the device: the
 *      histogram LocalTrajectoryBuilder3D::InsertIntoSubmap stores with every inserted node (LTB:605-610). points: n x 3 floats,
 *      already rotated by the node's gravity alignment. Float sums keep the reference's order; atan2f is the device's, so the
 *      result agrees with the CPU to float tolerance, not bit for bit. size <= 1024. ------------------------------------------ */
int dl_rotational_histogram(dl_context* ctx, const float* points, int64_t n, int32_t size, float* histogram_out);

/* ---- mapping::LocalTrajectoryBuilder3D (C/mapping/internal/3d/local_trajectory_builder_3d.h:81-113): the per-trajectory front-end
 *      object. AddImuData / AddRangeData -> MatchingResult{time, local_pose, range_data_in_local, InsertionResult}. Behind it:
 *      the IMU-coupled front end above against the matching submap (active submaps' front, LTB:502-505), the motion filter
 *      (C/mapping/internal/motion_filter.cc:37-57), Submap3D::InsertRangeData into both active submaps and the submap hand-over
 *      (C/mapping/3d/submap_3d.cc:264-279, :300-326) on the DEVICE grids, and the rotational histogram of the inserted scan.
 *      Deliberate differences from the reference: the pose comes from the fused scan-match + IMU solve instead of the match
 *      followed by the GTSAM window (LTB:535-555); num_accumulated_range_data = 1; one range sensor per builder (several are
 *      merged on the host by dliom::sensor::RangeDataSynchronizer, host/dliom_b200.hpp); initialisation = InitializeStatic
 *      (LTB:203-229) or dl_ltb_set_initial_state instead of the PCL NDT variant. ------------------------------------------- */
typedef struct dl_local_trajectory_builder dl_local_trajectory_builder;
typedef struct dl_ltb_options { /* proto::LocalTrajectoryBuilderOptions3D, the fields this path reads */
  dl_frontend_options frontend;                    /* ranges, voxel filters, adaptive filters, ceres options, scan_period */
  dl_imu_noise imu_noise;                          /* imu_options: acc / gyr noise and bias random walk */
  double imu_weight;                               /* weight of the pre-integration residual in the fused solve */
  double gravity;                                  /* imu_options.gravity (9.8) */
  float high_resolution, low_resolution;           /* submaps: 0.1 / 0.45 */
  int32_t num_range_data;                          /* submaps.num_range_data */
  int32_t high_resolution_max_range;               /* submaps.high_resolution_max_range */
  dl_range_data_inserter_options range_data_inserter;
  double motion_filter_max_time_seconds, motion_filter_max_distance_meters, motion_filter_max_angle_radians;
  int32_t rotational_histogram_size;
  int32_t frames_for_static_initialization;        /* 7 in the reference (LTB:376) */
  /* 0: the fused solve (scan match + IMU residual in one problem) gives the node's state. 1: the reference's TWO-STAGE chain —
   * plain CeresScanMatcher3D::Match from the IMU-predicted pose (LTB:535-542), then the window update with that pose as a prior
   * (dl_window_optimize_batch; LTB:555, :693-863); the carried information starts from the reference's priors (LTB:84-90).
   * Both modes take frontend.use_online_correlative_scan_matching: the correlative pre-match (LTB:514-521) then seeds the
   * solve from its pose, the translation target staying the prediction's (LTB:536). frontend.ceres_scan_matcher
   * .only_optimize_yaw is taken by the two-stage chain's plain solve; dl_ltb_create refuses it for the fused solve. */
  int32_t two_stage;
  int32_t reserved;
  double ceres_pose_noise_t, ceres_pose_noise_r;   /* imu_options: sigmas of the matched pose in the window */
  double prior_pose_noise, prior_velocity_noise, prior_bias_noise; /* LTB:84-90: prior_pose_n, 1e4, 1e-2 */
} dl_ltb_options;
typedef struct dl_matching_result {
  int32_t has_result;                              /* 0 <=> the reference returns nullptr (initialising, no IMU yet, scan dropped) */
  int32_t inserted;                                /* 0 <=> insertion_result == nullptr (motion filter) */
  double time;
  double local_pose[7];
  dl_nav_state state;                              /* pose + velocity + biases of the node (the reference's prev_state_ / prev_bias_) */
  dl_scan_result scan;                             /* the front end's bookkeeping for this scan */
  float origin_in_local[3];                        /* range_data_in_local.origin */
  int32_t num_returns, num_misses, num_high_resolution, num_low_resolution;
  int32_t num_insertion_submaps;                   /* insertion_submaps, queried before the insert (LTB:592-597) */
  int32_t insertion_submap_index[2];
  int32_t reserved;
} dl_matching_result;
int dl_ltb_create(dl_context* ctx, const dl_ltb_options* options, dl_local_trajectory_builder** out);
void dl_ltb_destroy(dl_local_trajectory_builder* builder);
int dl_ltb_set_initial_state(dl_local_trajectory_builder* builder, const dl_nav_state* state);
int dl_ltb_add_imu_data(dl_local_trajectory_builder* builder, double time, const double* linear_acceleration,
                        const double* angular_velocity);
/* xyzt: n TimedPointCloud rows (x y z t, t <= 0 relative to `time`, the last point's acquisition); origin: 3 floats (tracking frame). */
int dl_ltb_add_range_data(dl_local_trajectory_builder* builder, double time, const float* xyzt, int64_t n, const float* origin,
                          dl_matching_result* result);
/* The same for the output of the range-data synchroniser (C/mapping/internal/3d/range_data_synchronizer.cc:29-117, kaist / viral
 * run two LiDARs): rows of row_floats floats — 8 = RangeMeasurement {x y z t, u64 origin index}, 4 = x y z t with one origin —
 * sorted by time, and one origin per sensor. */
int dl_ltb_add_synchronized_range_data(dl_local_trajectory_builder* builder, double time, const void* rows, int64_t n,
                                       int32_t row_floats, const float* origins, int32_t num_origins, dl_matching_result* result);
/* Several trajectories in one call: item k is the arguments of one dl_ltb_add_synchronized_range_data on items[k].builder, and
 * afterwards results[k] and everything observable on that builder (state, clouds, histogram, submaps and their grids' cells)
 * are byte for byte what that single call would have produced. Members are independent, so their order does not matter. The
 * scans of all members run through one front-end batch, each against its own builder's matching submap, and the insertions
 * into all their active submaps share one set of host steps: the host waits a fixed number of times per call whatever
 * `count` is, except once for each grid whose pools or top level have to grow and for each submap a member hands over to.
 * A member to which one of the single call's early returns applies (initialising, n == 0, no IMU since the last scan) takes
 * no part in the device work. Rules, checked before any builder is touched (DL_ERR_ARG, every builder unchanged):
 * one dl_context for all builders, no builder twice, and equal dl_ltb_options on every builder, field by field (the batched
 * front end takes one options block and one IMU noise). count == 0 is a no-op. Each builder's host state is committed
 * only after the call's device work has succeeded. A call that fails after its device work has begun (a CUDA error, out of
 * memory, a cloud the rotational histogram refuses — the latter is detected before any grid changes) commits no builder's host
 * state, but after a failure inside the insertion the grids of the members' active submaps may already hold their scans: do not
 * feed such a builder the same scan again. dl_ltb_add_range_data and dl_ltb_add_synchronized_range_data are the batch of one.
 * With use_online_correlative_scan_matching every member's scan is pre-matched against its own matching submap's
 * high-resolution grid in the batch's one scoring launch (a fixed number of extra host waits per call); dl_matching_result.scan.rtcsm_score
 * carries the score (0 when the pre-match is off). Where the reference CHECK-fails on a candidate whose score is not > 0
 * (real_time_correlative_scan_matcher_3d.cc:111), the call fails with DL_ERR_SCORE before any grid changes and commits no
 * builder. */
typedef struct dl_ltb_batch_item {
  dl_local_trajectory_builder* builder;
  double time;
  const void* rows;        /* as dl_ltb_add_synchronized_range_data: row_floats 4 (x y z t, one origin) or 8 (RangeMeasurement) */
  int64_t n;
  int32_t row_floats;
  int32_t num_origins;
  const float* origins;    /* num_origins x 3 */
} dl_ltb_batch_item;
int dl_ltb_add_range_data_batch(int32_t count, const dl_ltb_batch_item* items, dl_matching_result* results);
/* Clouds of the last scan that produced a result. which: 0 returns / 1 misses of range_data_in_local, 2 / 3 the high / low
 * resolution point clouds in the tracking frame (TrajectoryNode::Data). Pass out = NULL to query *num_points. */
int dl_ltb_get_cloud(const dl_local_trajectory_builder* builder, int32_t which, float* out, int64_t capacity_points, int64_t* num_points);
int dl_ltb_get_histogram(const dl_local_trajectory_builder* builder, float* out, int32_t capacity);
int32_t dl_ltb_num_submaps(const dl_local_trajectory_builder* builder);
/* Submap `index` (0 = the first ever created): its device grids (owned by the builder; NULL once released), local pose, insert
 * count, finished flag. */
int dl_ltb_get_submap(dl_local_trajectory_builder* builder, int32_t index, dl_grid** high_resolution_grid,
                      dl_grid** low_resolution_grid, double* local_pose, int32_t* num_range_data, int32_t* finished);
/* Frees the two device grids of finished submap `index` (the reference's shared_ptr<const Submap3D> dropping to zero once the
 * pose graph trimmed it); the record (local pose, insert count, finished flag) stays. An active submap, an unknown index or
 * a second release: DL_ERR_ARG, nothing freed. */
int dl_ltb_release_submap(dl_local_trajectory_builder* builder, int32_t index);
int dl_ltb_get_state(const dl_local_trajectory_builder* builder, dl_nav_state* state, int32_t* initialized);

/* ---- submap images: Submap3D::ToResponseProto's X-ray textures (C/mapping/3d/submap_3d.cc:53-178, :253-262) and the fork's
 *      ProjectToCvMat (:381-464), the 8-bit image the loop detector's feature stage reads, computed on the device from the grids
 *      in place, for any number of (grid, pose) queries per call (each its own grid and pose; a grid may appear many times).
 *      Both walk every cell HybridGrid::Iterator yields (value != 0), skip it when ValueToProbability(value) < 0.501f, move the
 *      cell centre index * resolution by a Rigid3f and take lround(c * (1.f / resolution)) per axis (ExtractVoxelData,
 *      :82-112). Per pixel (x, y): the cell count, min / max z, the largest probability (from 0.5f) and the float sum of the
 *      probabilities in iterator order — lexicographic in (z/64, y/64, x/64, z/8 % 8, y/8 % 8, x/8 % 8, z % 8, y % 8, x % 8),
 *      as dl_grid_export_cells emits the cells.
 *   Textures (AddToTextureProto): the transform is pose.cast<float>() (the submap's global pose); width = max_y - min_y + 1,
 *      height = max_x - min_x + 1; cell (x, y) goes to pixel (max_x - x) * width + (max_y - y), two bytes (value, alpha) each,
 *      ComputePixelValues (:116-146) exactly, ProbabilityToLogOddsInteger's logf included (a host-built table of its steps).
 *      slice_pose = pose.inverse() * Translation(max_x * resolution, max_y * resolution, pose z), the two products in float.
 *   Projections (ProjectToCvMat): the transform is the pose's rotation without its yaw: Embed3D(Rigid2d::Rotation(-GetYaw))
 *      .cast<float>() * Rigid3d::Rotation(q).cast<float>() (:385-390, built on the host); width = max_x - min_x + 1, height =
 *      max_y - min_y + 1, row-major, pixel (y - min_y) * width + (x - min_x) = (uint8) lround((sum - 0.1f) * (255.f / 0.8f)) for
 *      every pixel: an empty pixel is 224, and the int -> uchar conversion wraps dense columns, as the reference does.
 *      ox = min_x * (double)resolution, oy = min_y * (double)resolution. Pass the submap's LOCAL pose for the loop detector
 *      (pose_graph_3d.cc:1078-1096 via ConstraintBuilder3D::ExtractFeaturesForSubmap).
 * Deliberate differences:
 *   - the texture's cells are returned raw, not through common::FastGzipString: compress them if a SubmapQuery needs it;
 *   - the fork's cv::threshold / cv::erode after ProjectToCvMat are not applied (OpenCV, host, cheap on the 8-bit image);
 *   - a grid without an obstructed cell (empty included) gives width = height = 0 and slice_pose / ox / oy all 0, where the
 *     reference's bounding box is INT_MIN - INT_MAX (undefined behaviour).
 * Pass cells / pixels = NULL to fill the per-query records and *num_bytes only (the images' bytes at each record's `offset`);
 * otherwise `capacity` must be at least *num_bytes. Grids are read only; they must be synced (dl_grid_sync after
 * dl_grid_set_cells) and not modified during the call. The host waits three times per call (two when sizing), whatever the
 * query count, plus once when the context's device scratch has to grow; the grids' pool sizes are read with one 8-byte copy per
 * query, the kernel launches do not depend on the query count. The size query runs the whole cell pass once, so sizing and then
 * filling reads every cell three times. Fails with DL_ERR_ARG while a dl_frontend_submit batch is in flight on `ctx`. */
typedef struct dl_submap_image_query {
  const dl_grid* grid;
  double pose[7];
} dl_submap_image_query;
typedef struct dl_submap_texture {
  float resolution;
  int32_t width, height;
  int32_t reserved;
  double slice_pose[7];
  int64_t offset;  /* first byte of the 2 * width * height interleaved (value, alpha) bytes */
} dl_submap_texture;
typedef struct dl_submap_projection {
  float resolution;
  int32_t width, height;
  int32_t reserved;
  double ox, oy;
  int64_t offset;  /* first byte of the width * height pixels */
} dl_submap_projection;
int dl_submap_textures(dl_context* ctx, int32_t count, const dl_submap_image_query* queries, dl_submap_texture* textures,
                       int64_t capacity, uint8_t* cells, int64_t* num_bytes);
int dl_submap_projections(dl_context* ctx, int32_t count, const dl_submap_image_query* queries, dl_submap_projection* projections,
                          int64_t capacity, uint8_t* pixels, int64_t* num_bytes);

/* ---- map writer: the assets writer's point pipeline for a finished run (cartographer_ros/assets_writer.cc:120-160 HandleMessage,
 *      the fork's config dlio/config/assets_writer_tongji.lua) on the device. Per message (one io::PointsBatch):
 *        point time = stamp + FromSeconds(t) (ticks of 100 ns, truncated toward zero), a point with !Has(time) is dropped
 *        (transform_interpolation_buffer.cc:45-66, Interpolate in timestamped_transform.cc:22-37: fp64 lerp + Eigen slerp),
 *        sensor_to_map = (tracking_to_map(time) * sensor_to_tracking).cast<float>(), output point = sensor_to_map * p, the batch
 *        origin = the translation of the last kept point's sensor_to_map; a message without a kept point makes no batch;
 *      then, in this fixed order:
 *        min_max_range_filter (io/min_max_range_filtering_points_processor.cc): keep iff min_range <= |p - origin| <= max_range,
 *          the float norm compared in double;
 *        voxel_filter_and_remove_moving_objects (io/outlier_removing_points_processor.cc), three passes over the whole input:
 *          pass 1 counts hits per cell (lround(p / (float)voxel_size)), pass 2 walks every ray from the batch origin in steps of
 *          voxel_size (for (float x = 0; x < length; x += voxel_size)) and adds one ray to the sample's cell if it has hits,
 *          pass 3 removes a point iff !(rays < 3 * hits) of its cell. Hits and rays are integer counts (no float atomics), so
 *          they do not depend on the order of the work.
 *      Restart protocol (PointsProcessor::FlushResult): stream every message of every trajectory through
 *      dl_map_writer_process(_dev), then call dl_map_writer_flush; if *restart is 1 (twice with moving-object removal), stream
 *      all of it again. Output points come only from the final pass. Node times are universal ticks (100 ns, the value of
 *      proto::Trajectory::Node::timestamp) and must be non-decreasing; trajectories are added before the first process call.
 *      Rejected with DL_ERR_ARG, the writer unchanged: an unknown trajectory, a trajectory added twice or after processing began,
 *      rows outside [0, num_rows), a call after the final flush, and (pass 1) a kept point whose cell lies beyond the hybrid
 *      grid's largest extent, +-8192 cells per axis (the reference's grid CHECK-fails there, hybrid_grid.h:391), or whose batch
 *      origin's cell does (a ray that long could stall pass 2's float step, where the reference loops forever).
 *      X-ray images (io/xray_points_processor.cc) and color_points (io/coloring_points_processor.cc) of the final pass's points,
 *      see dl_map_writer_add_xray. 2D occupancy grids of the final pass (io/probability_grid_points_processor.cc,
 *      cartographer_ros/ros_map_writing_points_processor.cc), see dl_map_writer_add_probability_grid. Not built: intensities,
 *      write_hybrid_grid, write_ply / write_xyz, the fixed-ratio sampler, frame-id filters, bag / tf reading. ---- */
typedef struct dl_map_writer dl_map_writer;
typedef struct dl_map_writer_options {
  int32_t range_filter;        /* 1: min_max_range_filter is in the pipeline */
  int32_t reserved;
  double min_range, max_range;
  double outlier_voxel_size;   /* > 0: voxel_filter_and_remove_moving_objects is in the pipeline, with this voxel_size */
} dl_map_writer_options;
typedef struct dl_map_message {  /* one PointsBatch: rows [first_row, first_row + num_rows) of the call's x y z t rows */
  int64_t stamp;                 /* universal ticks of the message (the time the row times t, in seconds, are relative to) */
  int64_t first_row, num_rows;
  int32_t trajectory_id;
  int32_t frame_id;              /* caller-chosen integer for PointsBatch::frame_id; only colour stages read it */
  double sensor_to_tracking[7];
} dl_map_message;
typedef struct dl_map_writer_info {  /* of one process call */
  int32_t pass;                      /* 0, 1 or 2: the pass this call belonged to */
  int32_t final_pass;                /* 1 if this pass produces the output points */
  int64_t num_rows;                  /* rows of the call's messages */
  int64_t dropped_no_pose;           /* !Has(time) */
  int64_t dropped_range;             /* min_max_range_filter */
  int64_t dropped_moving;            /* moving-object removal (final pass only) */
  int64_t messages_without_batch;
  int64_t num_samples;               /* pass 2: ray samples taken */
  int64_t num_points_out;
} dl_map_writer_info;
int dl_map_writer_create(dl_context* ctx, const dl_map_writer_options* options, dl_map_writer** out);
void dl_map_writer_destroy(dl_map_writer* writer);
/* times: num_nodes universal ticks (non-decreasing), poses: 7 doubles per node (the node's global pose). */
int dl_map_writer_add_trajectory(dl_map_writer* writer, int32_t trajectory_id, int32_t num_nodes, const int64_t* times,
                                 const double* poses);
/* xyzt_rows: num_rows rows of x y z t floats (sensor frame, t in seconds relative to the message stamp, e.g. the rows of
 * dl_decode_point_cloud2 with an identity sensor_to_tracking). points_out: room for as many x y z points as the messages have
 * rows (may be NULL when the call is not in the final pass). origins_out (optional): 3 floats per message, the batch origin, NaN
 * for a message without a batch. info may be NULL. At most 2^31 - 1 message rows per call. */
int dl_map_writer_process(dl_map_writer* writer, int32_t num_messages, const dl_map_message* messages, const float* xyzt_rows,
                          int64_t num_rows, float* points_out, int64_t* num_points_out, float* origins_out,
                          dl_map_writer_info* info);
/* The same with device rows in and device points out (16-byte aligned rows, as dl_decode_point_cloud2_dev writes them). */
int dl_map_writer_process_dev(dl_map_writer* writer, int32_t num_messages, const dl_map_message* messages,
                              const float* xyzt_rows_dev, int64_t num_rows, float* points_out_dev, int64_t* num_points_out,
                              float* origins_out, dl_map_writer_info* info);
/* Ends a pass: *restart = 1 if every message must be streamed again, 0 when the final pass ended (the writer is then finished). */
int dl_map_writer_flush(dl_map_writer* writer, int32_t* restart);
/* The moving-object removal's cell table, sorted by cell index (x, then y, then z): 3 ints per cell, hits, rays. Pass
 * cells_xyz = NULL to query *count. */
int dl_map_writer_voxels(const dl_map_writer* writer, int64_t capacity, int32_t* cells_xyz, int32_t* hits, int32_t* rays,
                         int64_t* count);

/* ---- X-ray images and point colours of the final pass (io/xray_points_processor.cc, io/coloring_points_processor.cc).
 *      Stages are added after create and before the first process call, in pipeline order, and sit after the last multi-pass
 *      stage: they see exactly the final pass's output points, messages in call order, rows in message order (the reference
 *      LOG(FATAL)s when X-ray generation comes before a multi-pass stage). At most DL_MAP_WRITER_MAX_STAGES stages of both
 *      kinds together.
 *        color_points: a message whose frame_id equals the stage's gets every point coloured rgb[i] / 255.f. An X-ray stage sees
 *          the colour stages added before it, the last matching one wins; a message none of them touched has no colours and adds
 *          kDefaultColor (0, 0, 0).
 *        write_xray_image: camera_point = transform.cast<float>() * p, cell = lround(camera_point / (float)voxel_size) per axis;
 *          the cell becomes occupied, extends the bounding box, and its column (y, z) adds the colour to float sums in stream
 *          order and counts the point. The image is (max.y - min.y + 1) x (max.z - min.z + 1), cell (y, z) at pixel
 *          (max.y - y, max.z - z); a pixel mixes white with the column's mean colour by log(occupied voxels) / max over columns
 *          of that log (IntoImage, including its double / float promotions); an empty column is white. Images equal the
 *          reference's with draw_trajectories = false (trajectory strokes are Cairo's antialiasing and are not drawn).
 *      Rejected with DL_ERR_ARG, the writer unchanged: a stage added after processing began or beyond the cap, voxel_size <= 0 or
 *      not finite, a quaternion with |norm - 1| > 1e-9 (FromDictionary's CHECK_NEAR), and (final pass) a point whose X-ray cell
 *      lies beyond +-8192 on any axis (where HybridGridBase<bool>::mutable_value CHECK-fails). ---- */
#define DL_MAP_WRITER_MAX_STAGES 16
typedef struct dl_map_writer_color {
  int32_t frame_id;
  uint8_t rgb[3];                /* the Lua values after static_cast<uint8> */
  uint8_t pad;
} dl_map_writer_color;
typedef struct dl_map_writer_xray {
  double voxel_size;
  double transform[7];           /* Rigid3d: t x y z, q w x y z */
} dl_map_writer_xray;
int dl_map_writer_add_color(dl_map_writer* writer, const dl_map_writer_color* color);
/* *stage receives the X-ray stage's number (0, 1, ... in the order X-ray stages were added). */
int dl_map_writer_add_xray(dl_map_writer* writer, const dl_map_writer_xray* xray, int32_t* stage);
/* After the final flush: the image of an X-ray stage as Cairo ARGB32 words 0xFF000000 | r << 16 | g << 8 | b, row-major,
 * *width * *height of them. Pass argb = NULL to query the size; capacity is in words. An empty bounding box gives 0 x 0 (the
 * reference writes no file then). Rejected with DL_ERR_ARG: an unknown stage, a call before the final flush, capacity too small. */
int dl_map_writer_xray_image(const dl_map_writer* writer, int32_t stage, int64_t capacity, uint32_t* argb, int32_t* width,
                             int32_t* height);

/* ---- 2D occupancy grids of the final pass: write_probability_grid (io/probability_grid_points_processor.cc) and write_ros_map
 *      (cartographer_ros/ros_map_writing_points_processor.cc) share this stage. Added like an X-ray stage (after create, before
 *      the first process call, counted against DL_MAP_WRITER_MAX_STAGES with the other kinds); several may coexist.
 *      Every batch of the final pass (a message whose origin is not NaN, also when the range filter or the moving-object
 *      removal emptied it) is one ProbabilityGridRangeDataInserter2D::Insert({origin, points, {}}): only x and y are used.
 *        the grid starts as CreateProbabilityGrid(resolution): 100 x 100 cells, max = 50 * resolution per axis (double);
 *        GrowAsNeeded: the float box of the origin and the points, GrowLimits(min - 1e-6f) and GrowLimits(max + 1e-6f), each
 *          doubling both axes around the centre until the cell is contained (grid_2d.cc:116);
 *        GetCellIndex(p) = (lround((max.y - p.y) / res - 0.5), lround((max.x - p.x) / res - 0.5)) in double;
 *        CastRays at res / 1000 (ray_casting.cc:166): the hit table on every point's cell, then (insert_free_space) the
 *          subpixel walk CastRay(origin, point) with the miss table; a cell is updated at most once per batch and a hit wins over
 *          any miss (kUpdateMarker). The tables are ComputeLookupTableToApplyCorrespondenceCostOdds(Odds((float)p)).
 *      Rejected with DL_ERR_ARG, the writer unchanged: a stage added after processing began or beyond the cap, a resolution <= 0
 *      or not finite, hit_probability <= 0.5 or miss_probability >= 0.5 (the reference's CHECKs) or either not finite, and (final
 *      pass) a point whose x or y is not finite or a batch whose growth would take a grid beyond DL_MAP_WRITER_MAX_GRID_CELLS
 *      cells per axis (the reference's superscaled num_cells * 1000 must fit an int). A failed allocation returns DL_ERR_CUDA,
 *      the writer unchanged. A writer returns the same points, origins and info with or without grid stages. ---- */
#define DL_MAP_WRITER_MAX_GRID_CELLS (100 << 14)
typedef struct dl_map_writer_grid_options {
  double resolution;
  double hit_probability, miss_probability;  /* range_data_inserter: > 0.5 and < 0.5 */
  int32_t insert_free_space;                 /* 1 (the reference's default) or 0 */
  int32_t reserved;
} dl_map_writer_grid_options;
typedef struct dl_map_writer_grid_info {
  double resolution, max_x, max_y;           /* MapLimits after the final flush */
  int32_t num_x_cells, num_y_cells;
  int32_t offset_x, offset_y;                /* ComputeCroppedLimits: the known-cells box, or 0, 0 and 1 x 1 when it is empty */
  int32_t width, height;                     /* cropped num_x_cells, num_y_cells */
} dl_map_writer_grid_info;
/* *stage receives the grid stage's number (0, 1, ... in the order grid stages were added). */
int dl_map_writer_add_probability_grid(dl_map_writer* writer, const dl_map_writer_grid_options* options, int32_t* stage);
/* After the final flush: the grid's limits and cropped box in *info; cells (optional) receives the Grid2D uint16 correspondence-cost
 * values of the cropped box, row-major (cell (offset_x + x, offset_y + y) at y * width + x, 0 = unknown); pixels (optional)
 * receives DrawProbabilityGrid's grey values of the same box, unrotated (128 for an unknown cell, else
 * lround(255 * (((1 - p) - 0.1f) / ((1 - 0.1f) - 0.1f))) in float). Both NULL queries the size; capacity is in cells. Rejected with
 * DL_ERR_ARG: an unknown stage, a call before the final flush, capacity below width * height. */
int dl_map_writer_probability_grid(const dl_map_writer* writer, int32_t stage, dl_map_writer_grid_info* info, int64_t capacity,
                                   uint16_t* cells, uint8_t* pixels);

/* Device memory helpers so a host language without CUDA bindings can stage buffers. */
int dl_device_alloc(dl_context* ctx, int64_t bytes, void** out_dev);
int dl_device_free(dl_context* ctx, void* dev);
int dl_copy_to_device(dl_context* ctx, void* dst_dev, const void* src_host, int64_t bytes);
int dl_copy_to_host(dl_context* ctx, void* dst_host, const void* src_dev, int64_t bytes);

#ifdef __cplusplus
}
#endif
#endif /* DLIOM_B200_H_ */
