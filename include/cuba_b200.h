/*
 * cuba_b200.h -- C ABI of the H100-native Levenberg-Marquardt bundle-adjustment engine.
 *
 * This is the drop-in boundary for the ONE hot path of fixstars/cuda-bundle-adjustment:
 * everything the reference's CudaBlockSolver does below `optimize()` (paths relative to the reference
 * checkout):
 *
 *   what this ABI replaces                                   reference interface
 *   ------------------------------------------------------   -------------------------------------------------
 *   cuba_engine_set_problem   (flat arrays -> device, + all   CudaBlockSolver::initialize/buildStructure,
 *                              sparsity structures)           src/cuda_bundle_adjustment.cpp:115-366;
 *                                                             gpu::buildHplStructure / findHschureMulBlockIndices,
 *                                                             src/cuda_block_solver.h:36-41;
 *                                                             HschurSparseBlockMatrix, src/sparse_block_matrix.h:81-98
 *   cuba_engine_optimize      (whole LM loop)                 CudaBundleAdjustmentImpl::optimize, cpp:793-857
 *   cuba_stage_linearize      (residual+Jacobian+Hessian)     gpu::computeActiveErrors + gpu::constructQuadraticForm,
 *                                                             src/cuda_block_solver.h:43-57
 *   cuba_stage_max_diagonal                                   gpu::maxDiagonal, h:65-67
 *   cuba_stage_solve          (Schur + PCG + back-subst.)     gpu::addLambda/computeBschure/computeHschure/
 *                                                             convertHschureBSRToCSR/schurComplementPost, h:69-88 and
 *                                                             SparseLinearSolver::solve, src/cuda_linear_solver.h:28-39
 *   cuba_stage_update         (SE3 exp update + trial chi2)   gpu::updatePoses/updateLandmarks/computeScale, h:90-94
 *   cuba_engine_get_state / _get_chi2 / _get_profile          CudaBlockSolver::finalize/getChiSqs/getTimeProfile,
 *                                                             cpp:512-562
 *
 * Plain C types only: pointers and sizes, no torch / Eigen / STL types.  All host arrays are fp64 and
 * column-major where they hold blocks (reference MatView, src/cuda_block_solver.cu:79-85); an engine
 * configured for fp32 narrows at this boundary like the reference's ScalarCast (cpp:54-69).
 *
 * Every function returns CUBA_OK (0) or a negative error code; cuba_last_error() gives the message.
 * The library has NO CPU fallback: without a usable CUDA device every compute entry point fails with
 * CUBA_ERR_CUDA.
 */
#ifndef CUBA_B200_H
#define CUBA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CUBA_OK 0
#define CUBA_ERR_INVALID (-1)  /* bad argument / inconsistent problem                */
#define CUBA_ERR_CUDA (-2)     /* CUDA runtime failure or no device                  */
#define CUBA_ERR_STATE (-3)    /* call order violated (e.g. optimize before problem) */
#define CUBA_ERR_COMM (-4)     /* NCCL failure                                       */

/* robust kernels: reference include/cuda_bundle_adjustment_types.h:213-218, cu:692-727 */
#define CUBA_ROBUST_NONE 0
#define CUBA_ROBUST_HUBER 1
#define CUBA_ROBUST_TUKEY 2

/* edge types: reference include/cuda_bundle_adjustment_types.h:143-148 */
#define CUBA_EDGE_MONOCULAR 0
#define CUBA_EDGE_STEREO 1

/* time-profile buckets: same 8 items as the reference, cpp:77-88,547-557 */
#define CUBA_PROF_INITIALIZE 0
#define CUBA_PROF_BUILD_STRUCTURE 1
#define CUBA_PROF_COMPUTE_ERROR 2
#define CUBA_PROF_BUILD_SYSTEM 3
#define CUBA_PROF_SCHUR_COMPLEMENT 4
#define CUBA_PROF_DECOMP_SYMBOLIC 5   /* always 0: PCG has no symbolic phase */
#define CUBA_PROF_DECOMP_NUMERICAL 6  /* the PCG solve, or the dense Cholesky  */
#define CUBA_PROF_UPDATE 7
#define CUBA_PROF_NUM 8

typedef struct cuba_config {
	int device;            /* CUDA device ordinal, -1 = current device                            */
	int use_fp32;          /* 0 = fp64 (default); 1 = reference's USE_FLOAT32 behaviour; 2 = mixed precision: fp64 engine whose Hpl
	                          blocks -- the dominant 144 B/edge stream -- are STORED in fp32 (80-byte blocks), everything computed
	                          and accumulated in fp64, PCG in fp64 (SURVEY.md 8 f-4)                                        */
	int pcg_max_iters;     /* <=0: default (see DESIGN.md)                                         */
	double pcg_tol;        /* stop when sqrt(r'z / r0'z0) <= pcg_tol; <=0: default 1e-11 (fp64)    */
	int deterministic;     /* kept for layout compatibility; every kernel sums in a fixed order: results are bit-reproducible run to run */
	int reserved[7];       /* reserved[0]: reduced-system solver.  0 (default) = automatic: block-Jacobi PCG while a solve converges within
	                          reserved[5] iterations (k_pcg3 on one GPU: shared-memory resident, flag-synchronised exchange, no barrier
	                          in the iteration), two-level PCG afterwards (k_pcg5, cuba_pcg5.cuh: block-Jacobi + coarse correction
	                          over rigid motions of pose aggregates in the same flag-synchronised protocol).  With several ranks and
	                          >= 2048 free poses k_pcg5 runs with the block rows DISTRIBUTED over the ranks (NVLink peer boards);
	                          7 = never distribute (replicated solve), 8 = always distribute.  5 = always two-level k_pcg5,
	                          6 = always block-Jacobi k_pcg5, 3 = always k_pcg4 (two-level, one grid barrier per iteration),
	                          4 = always k_pcg3, 2 = k_pcg2 (one grid barrier per iteration).  A solve the chosen kernel cannot
	                          take runs block-Jacobi k_pcg3 (k_pcg2 beyond its rows per CTA)
	                          reserved[1]: 1 = build the index structures on the host (cuba_structure.cpp) instead of
	                          on the device (cuba_structure_gpu.cuh, default); both give identical structures
	                          reserved[2]: J+H landmark kernel, 0 = k_linearize_landmark4 (warp tiles, default; 8/9 = 5/6 CTAs per SM,
	                          7 = three pipeline stages), 1-4 = first generation (tile shapes; the fp32 engine's kernel)
	                          reserved[3]: Schur kernel, 0 / 3 = k_schur3 (six lanes per product, default), 5 = landmark tiles on the
	                          fp64 tensor pipe (cuba_schur5.cuh, DMMA m8n8k4; wins only on banded graphs; k_schur3 where it cannot run:
	                          fp32 or mixed precision, host-built structures, and a graph with a repeated (pose, landmark) pair)
	                          reserved[0], [2] and [3] accept only the values listed: cuba_engine_create returns CUBA_ERR_INVALID
	                          for any other, before it touches a device
	                          reserved[4]: two-level PCG: solves between rebuilds of the coarse matrix (<=0: 8)
	                          reserved[5]: automatic solver: block-Jacobi iteration count that switches to two-level (<=0: 100)
	                          reserved[6]: two-level PCG: upper bound on the number of pose aggregates (<=0: 74; <= 37 uses the one-CTA inverse) */
} cuba_config;

/* Flat problem: exactly what CudaBlockSolver::initialize produces (cpp:115-261).
 * Vertices are indexed by iP / iL: free vertices first (iP < numP, iL < numL), fixed ones appended.
 * Edges with both ends fixed must not be present.  Edge ids: monocular 0..E2-1, stereo E2..E2+E3-1. */
typedef struct cuba_problem {
	int32_t Pall, numP;
	int32_t Lall, numL;
	const double* q;       /* [4*Pall] unit quaternions, coefficient order x,y,z,w                */
	const double* t;       /* [3*Pall]                                                            */
	const double* cam;     /* [5*Pall] fx,fy,cx,cy,bf per pose                                    */
	const double* Xw;      /* [3*Lall]                                                            */
	int32_t E2;
	const int32_t* idx2;   /* [2*E2] (iP,iL) per monocular edge                                   */
	const double* meas2;   /* [2*E2] (u,v)                                                        */
	const double* omega2;  /* [E2] scalar information                                             */
	int32_t E3;
	const int32_t* idx3;   /* [2*E3]                                                              */
	const double* meas3;   /* [3*E3] (u_left, v, u_right)                                         */
	const double* omega3;  /* [E3]                                                                */
} cuba_problem;

/* reference BatchInfo (include/cuda_bundle_adjustment_types.h:226-232) plus solver diagnostics */
typedef struct cuba_iter_stat {
	int32_t iteration;
	int32_t trials;        /* LM trials spent in this outer iteration (1 = first trial accepted)   */
	double chi2;           /* objective after the iteration (robustified, like the reference)      */
	double lambda;         /* damping after the iteration                                          */
	int32_t pcg_iters;     /* PCG iterations summed over the trials                                */
	int32_t pcg_failed;    /* number of trials whose PCG did not converge / broke down             */
} cuba_iter_stat;

typedef struct cuba_sizes {
	int32_t Pall, numP, Lall, numL, E2, E3;
	int32_t nhpl;          /* free-free edges = Hpl blocks                                         */
	int32_t nblk;          /* upper-triangular Hsc blocks                                          */
	int32_t nmul;          /* Schur block products                                                 */
	int32_t nblk_full;     /* blocks of the symmetric-full BSR used by the PCG                     */
} cuba_sizes;

typedef struct cuba_engine cuba_engine;

const char* cuba_last_error(void);
int cuba_version(void);

int cuba_engine_create(const cuba_config* cfg /* NULL = defaults */, cuba_engine** out);
int cuba_engine_destroy(cuba_engine* e);

/* setRobustKernels (include/cuda_bundle_adjustment.h:93): one kernel per edge type */
int cuba_engine_set_robust_kernel(cuba_engine* e, int edge_type, int kernel_type, double delta);

/* Landmark sharding for multi-GPU runs (one process per GPU).  Must precede set_problem.
 * `nccl_unique_id` = 128 bytes produced by cuba_comm_unique_id() on rank 0 and broadcast by the host
 * (torch.distributed / MPI / a file).  world == 1 disables it. */
int cuba_comm_unique_id(void* out128);
int cuba_engine_set_comm(cuba_engine* e, int rank, int world, const void* nccl_unique_id);

/* Upload the problem and build every index structure (initialize + buildStructure). */
int cuba_engine_set_problem(cuba_engine* e, const cuba_problem* p);
/* Linear solver of the reduced camera system S xp = bsc (S = Hsc + lambda I), g2o's choice of LinearSolver / Ceres' DENSE_SCHUR
 * vs ITERATIVE_SCHUR.  CUBA_SOLVER_PCG (default): the PCG family that cuba_config.reserved[0] selects.  CUBA_SOLVER_DENSE_CHOLESKY: a
 * dense fp64 Cholesky factorisation of S on the tensor pipe (csrc/cuba_dense_chol.cuh; the fp32 engine widens S), with the reference's
 * semantics: an exact step, and a trial whose factorisation fails (S not positive definite) is rejected.  It needs no PCG partition,
 * so graphs whose need lists do not fit the PCG's shared memory are accepted, and it takes at most 2730 free poses (n <= 16380,
 * about 1.1 GB of fp64 tiles): set_problem returns CUBA_ERR_INVALID beyond that, before any allocation, and the engine keeps its
 * previous problem.  A problem without free landmarks has no reduced camera system (its poses are solved block by block): there
 * the choice changes nothing, and neither the cap nor the tiles apply.  The choice applies from the next set_problem (a structure-reuse set_problem after a change rebuilds what the new
 * solver needs); any other value gives CUBA_ERR_INVALID. */
#define CUBA_SOLVER_PCG 0
#define CUBA_SOLVER_DENSE_CHOLESKY 1
int cuba_engine_set_linear_solver(cuba_engine* e, int solver);
/* Structure reuse (SURVEY.md 8 f-2; on by default): a set_problem whose sizes, fixed/free split and (iP,iL) lists equal those of the
 * problem the engine already holds keeps every device structure (index lists, tiles, product lists, PCG partition) and only
 * uploads the numbers -- repeated local-BA calls on an unchanged graph, e.g. the reference protocol's second initialize()
 * (samples/sample_ba_from_file.cpp:159-161).  The reference rebuilds everything (cpp:263-366).  Results are identical either way. */
int cuba_engine_set_structure_reuse(cuba_engine* e, int enable);
int cuba_engine_get_structure_reuses(cuba_engine* e, long long* count);
/* Replace only the estimate (q,t,Xw), keeping structure -- repeated optimize() on the same graph. */
int cuba_engine_set_state(cuba_engine* e, const double* q, const double* t, const double* Xw);

/* Restore the estimate last given by set_problem / set_state from its device-resident copy (no host
 * traffic): lets a benchmark time optimize() repeatedly with all inputs already in HBM. */
int cuba_engine_reset_state(cuba_engine* e);

int cuba_engine_get_sizes(const cuba_engine* e, cuba_sizes* out);
/* The CUDA stream (cudaStream_t) every kernel of this engine is launched on -- for CUDA-event timing. */
int cuba_engine_get_stream(cuba_engine* e, void** stream);
/* Overwrite a buffer larger than L2 on the engine's stream (benchmark hygiene between timed steps). */
int cuba_engine_flush_l2(cuba_engine* e);

/* optimize(niterations): stats[niterations]; *nstats = number of entries written (cpp:848-851). */
int cuba_engine_optimize(cuba_engine* e, int niterations, cuba_iter_stat* stats, int* nstats);

/* finalize(): current estimate, [4*Pall], [3*Pall], [3*Lall]; any pointer may be NULL */
int cuba_engine_get_state(cuba_engine* e, double* q, double* t, double* Xw);
/* getChiSqs(): non-robust omega*|r|^2 per edge, edge-id order, [E2+E3] */
int cuba_engine_get_chi2(cuba_engine* e, double* per_edge);
/* Edge levels (g2o Edge::setLevel + initializeOptimization(0)).  levels[E2+E3] in edge-id order; 0 = optimised, anything else =
 * kept in the problem but left out of the objective and the normal equations (and out of the chi2 of cuba_iter_stat).  NULL = all 0.
 * set_problem resets every level to 0; set_state, reset_state and optimize keep them.  Changing a level keeps the estimate and
 * drops what earlier solves left behind (the two-level PCG's coarse matrix).  The result is bit for bit that of a set_problem
 * whose omega is 0 on the edges at level 1.  get_chi2 still reports omega*|r|^2 with the caller's omega for every edge.  With no
 * edge at level 0, optimize() writes no iteration (*nstats = 0) and leaves the estimate alone.  Landmark-sharded runs: every rank
 * gets the same full array and applies its own edges. */
int cuba_engine_set_edge_levels(cuba_engine* e, const uint8_t* levels);
int cuba_engine_get_edge_levels(cuba_engine* e, uint8_t* levels);          /* 0 or 1 per edge */

/* The outlier test of ORB-SLAM2's local BA / pose optimisation, on the device, against the current estimate: an edge fails when its
 * non-robust omega*|r|^2 (the value get_chi2 returns) exceeds chi2_mono / chi2_stereo, or, with CUBA_CLASSIFY_DEPTH, when Xc.z <= 0.
 * Failing edges go to level 1.  Without CUBA_CLASSIFY_REINCLUDE, levels only go 0 -> 1 (local BA).  With it, an edge that passes goes
 * back to 0 (pose optimisation).  counts[4] (may be NULL): included mono, included stereo, newly excluded, re-included (summed over
 * the ranks).  One 32-byte read-back is the only host synchronisation. */
#define CUBA_CLASSIFY_DEPTH 1
#define CUBA_CLASSIFY_REINCLUDE 2
int cuba_engine_classify_edges(cuba_engine* e, double chi2_mono, double chi2_stereo, int flags, int32_t* counts);

/* Pose optimisation of many frames (ORB-SLAM2's Optimizer::PoseOptimization, batched).  A frame is one free SE(3) pose and its
 * edges, each carrying its own world point, which is held fixed.  Host arrays, fp64; the edges of frame b are [ptr2[b], ptr2[b+1])
 * and [ptr3[b], ptr3[b+1]), ptr2[0] = ptr3[0] = 0, ptr2[B] = E2, ptr3[B] = E3.  Array pointers of an empty edge type may be NULL. */
typedef struct cuba_pose_batch {
	int32_t B, E2, E3;
	const double* q;       /* [4B] x,y,z,w                                                         */
	const double* t;       /* [3B]                                                                 */
	const double* cam;     /* [5B] fx,fy,cx,cy,bf                                                  */
	const int32_t* ptr2;   /* [B+1]                                                                */
	const double* X2;      /* [3*E2] world point of each monocular edge                            */
	const double* meas2;   /* [2*E2]                                                               */
	const double* omega2;  /* [E2]                                                                 */
	const int32_t* ptr3;   /* [B+1]                                                                */
	const double* X3;      /* [3*E3]                                                               */
	const double* meas3;   /* [3*E3]                                                               */
	const double* omega3;  /* [E3]                                                                 */
} cuba_pose_batch;

/* One round of the schedule: optimize(iterations) with the given robust kernels (meaning of cuba_engine_set_robust_kernel, indexed by
 * CUBA_EDGE_*), from the frame's input pose when restart != 0 (ORB-SLAM2 sets the estimate at the top of every round), else from the
 * previous round's result; then the outlier test of cuba_engine_classify_edges on the committed pose. */
#define CUBA_POSE_MAX_ROUNDS 8
typedef struct cuba_pose_round {
	int32_t iterations;
	int32_t kernel_type[2];
	double delta[2];
	int32_t restart;
	double chi2_mono, chi2_stereo;
	int32_t flags;         /* CUBA_CLASSIFY_DEPTH | CUBA_CLASSIFY_REINCLUDE                         */
} cuba_pose_round;

/* Runs the schedule on every frame: ONE kernel launch (one CTA per frame), one host->device and one device->host copy.  Every edge
 * starts at level 0.  Each frame's result is what the engine computes for the frame's sub-problem (set_problem with one free pose
 * and the edges' points as fixed landmarks; per round set_robust_kernel, set_state on restart, optimize(iterations), classify_edges),
 * always in fp64; it is bit-reproducible and independent of the other frames of the batch.  A round with no edge at level 0 writes no
 * iteration and leaves the pose alone.  Runs on the engine's device and stream, ignores set_comm, and neither reads nor changes the
 * engine's problem, state, levels or solver state.
 * Outputs: q_out [4B], t_out [3B]; levels_out [E2+E3] (mono then stereo, 0/1 after the last round); counts [B][nrounds][4] (as
 * classify_edges); stats [B][sum of iterations] (round r of frame b at b * sum + iterations of rounds < r, pcg fields 0); nstats
 * [B][nrounds] (iterations written per round).  Every output except q_out / t_out may be NULL.  B = 0 does nothing.
 * CUBA_ERR_INVALID, with nothing run, for a malformed batch or schedule (B < 0, ptr not starting at 0, decreasing or not ending at
 * the edge count, nrounds outside 1..CUBA_POSE_MAX_ROUNDS, negative iterations, an unknown kernel type or flag, a non-finite omega
 * or delta). */
int cuba_engine_optimize_poses(cuba_engine* e, const cuba_pose_batch* batch, int nrounds, const cuba_pose_round* rounds,
	double* q_out, double* t_out, uint8_t* levels_out, int32_t* counts, cuba_iter_stat* stats, int32_t* nstats);

/* Sim(3) alignment of many keyframe pairs (ORB-SLAM2's Optimizer::OptimizeSim3, batched).  Problem b is keyframes 1 and 2 and the
 * matched pairs [ptr[b], ptr[b+1]); ptr[0] = 0, ptr[B] = N.  Pair i: X1 (point of keyframe 1 in camera-1 coordinates), X2 (its match
 * in camera-2 coordinates), obs1 / obs2 (the keypoints in keyframes 1 / 2), omega1 / omega2 (scalar informations).  The unknown is
 * S12 = (R(q), t, s), S12 X = s R X + t.  Each pair gives two monocular edges, r12 = pi1(S12 X2) - obs1 and r21 = pi2(S12^-1 X1) -
 * obs2, pi(Y) = (fx Y.x / Y.z + cx, fy Y.y / Y.z + cy), each under a Huber kernel with delta = sqrt(chi2).  With fix_scale[b] != 0
 * the scale is held (s_out is s bit for bit).  Host arrays, fp64; pair arrays may be NULL when N = 0. */
typedef struct cuba_sim3_batch {
	int32_t B, N;
	const int32_t* ptr;        /* [B+1]                                                                */
	const double* q;           /* [4B] x,y,z,w                                                         */
	const double* t;           /* [3B]                                                                 */
	const double* s;           /* [B]  > 0                                                             */
	const double* cam1;        /* [4B] fx,fy,cx,cy of keyframe 1                                       */
	const double* cam2;        /* [4B] fx,fy,cx,cy of keyframe 2                                       */
	const int32_t* fix_scale;  /* [B], or NULL: scale free everywhere                                  */
	const double* X1;          /* [3N]                                                                 */
	const double* X2;          /* [3N]                                                                 */
	const double* obs1;        /* [2N]                                                                 */
	const double* obs2;        /* [2N]                                                                 */
	const double* omega1;      /* [N]                                                                  */
	const double* omega2;      /* [N]                                                                  */
} cuba_sim3_batch;

/* OptimizeSim3(pKF1, pKF2, matches, S12, th2, bFixScale): optimize(iterations); the pair test (a pair fails when either edge's
 * non-robust omega |r|^2 exceeds chi2; failed pairs go to level 1); with fewer than min_pairs pairs left, 0 inliers and S out = S in;
 * else optimize(iterations_bad if the test removed a pair, else iterations_good) over the pairs left and the test again.  The defaults
 * are ORB-SLAM2's: CUBA_SIM3_DEFAULT_*. */
#define CUBA_SIM3_DEFAULT_CHI2 10.0
#define CUBA_SIM3_DEFAULT_ITERATIONS 5
#define CUBA_SIM3_DEFAULT_ITERATIONS_BAD 10
#define CUBA_SIM3_DEFAULT_ITERATIONS_GOOD 5
#define CUBA_SIM3_DEFAULT_MIN_PAIRS 10
typedef struct cuba_sim3_params {
	double chi2;
	int32_t iterations, iterations_bad, iterations_good, min_pairs;
} cuba_sim3_params;

/* Runs the schedule on every problem: ONE kernel launch (one CTA per problem), one host->device and one device->host copy.  The LM
 * rules are those of cuba_engine_optimize (lambda from the largest of the 7 diagonal entries); the update is S <- Exp(xi) S, xi =
 * (omega, upsilon, sigma), with analytic Jacobians.  Always fp64; each problem's result is bit-reproducible and independent of the
 * other problems of the batch.  Runs on the engine's device and stream, ignores set_comm, and neither reads nor changes the engine's
 * problem, state, levels or solver state.
 * Outputs: q_out [4B], t_out [3B], s_out [B]; levels_out [N] (0/1 after the last test); ninliers [B]; stats [B][iterations +
 * max(iterations_bad, iterations_good)] (the second optimize of problem b from b * that + iterations, pcg fields 0); nstats [B][2]
 * (iterations written by each optimize).  Every output except q_out / t_out / s_out may be NULL.  B = 0 does nothing.
 * CUBA_ERR_INVALID, with nothing run, for B < 0, a malformed ptr, a non-finite input, s <= 0, negative iterations or min_pairs, or a
 * chi2 that is not finite and positive. */
int cuba_engine_optimize_sim3(cuba_engine* e, const cuba_sim3_batch* batch, const cuba_sim3_params* params, double* q_out, double* t_out,
	double* s_out, uint8_t* levels_out, int32_t* ninliers, cuba_iter_stat* stats, int32_t* nstats);

/* seconds per profile bucket accumulated since set_problem, [CUBA_PROF_NUM] */
int cuba_engine_get_profile(cuba_engine* e, double* seconds);
/* number of kernels this library launched since create (for bench.py's gpu_launches) */
int cuba_engine_get_launch_count(cuba_engine* e, long long* count);

/* cumulative host->device / device->host bytes copied by this thread's engines (for bench.py's e2e record) */
int cuba_get_transfer_bytes(long long* h2d, long long* d2h);

/* ---- stage-wise entry points (used by optimize(); exported for stage parity tests) ---- */
int cuba_stage_linearize(cuba_engine* e, double* chi2);
int cuba_stage_max_diagonal(cuba_engine* e, double* maxdiag);
/* Schur complement with damping lambda, PCG, back-substitution.  *ok = 0 when PCG failed. */
int cuba_stage_solve(cuba_engine* e, double lambda, int* pcg_iters, int* ok);
/* trial update into the spare state buffer + its chi2 and the LM scale (without the +1e-3) */
int cuba_stage_update(cuba_engine* e, double lambda, double* chi2_trial, double* scale);
/* accept (swap buffers) or reject (keep) the trial state */
int cuba_stage_commit(cuba_engine* e, int accept);
/* residual-only pass on the current state */
int cuba_stage_chi2(cuba_engine* e, double* chi2);

/* ---- debug getters (host copies; blocks column-major; any pointer may be NULL) ---- */
/* Hpl CSC sorted by (iL,iP): colPtr[numL+1], rowInd[nhpl], edge2Hpl[E2+E3] (-1 = no block) */
int cuba_debug_get_hpl_structure(cuba_engine* e, int32_t* colPtr, int32_t* rowInd, int32_t* edge2Hpl);
/* Hsc upper-triangular BSR: rowPtr[numP+1], colInd[nblk] */
int cuba_debug_get_hsc_structure(cuba_engine* e, int32_t* rowPtr, int32_t* colInd);
int cuba_debug_get_system(cuba_engine* e, double* Hpp /*36*numP*/, double* bp /*6*numP*/, double* Hll /*9*numL*/,
	double* bl /*3*numL*/, double* Hpl /*18*nhpl*/);
int cuba_debug_get_schur(cuba_engine* e, double* Hsc /*36*nblk, upper*/, double* bsc /*6*numP*/, double* invHll /*9*numL*/);
int cuba_debug_get_delta(cuba_engine* e, double* xp /*6*numP*/, double* xl /*3*numL*/);

/* What the last cuba_stage_solve (or the last trial of optimize) ran, for tests of the PCG and its two-level preconditioner.
 * info[CUBA_PCG_INFO_LEN]:
 *   0 kernel (CUBA_PCG_KERNEL_*)             1 two-level solve (0/1)
 *   2..8 the k_pcg5 plan (zeros without one): aggregates per CTA, G (CTAs), gs (CTAs per aggregate), A (aggregates; nc = 6A),
 *        maxRows (most rows of one CTA), capBlocks (blocks cached in shared memory per CTA), zhInSmem (Z^ rows in shared memory)
 *   9 coarse-inverse kernel of the last solve (CUBA_COARSE_KERNEL_*; NONE for a block-Jacobi solve)
 *  10 cInfo of the last k_pcg5 coarse rebuild (0 ok, 1 not positive definite; -1 none yet)
 *  11 status of the last PCG (0 converged, 1 iteration cap, 2 breakdown)     12 its iterations
 *  13 k_pcg5 coarse rebuilds since set_problem                                14 block-Jacobi retries of optimize() since set_problem
 *  15 of the last 256 k_pcg5 coarse rebuilds, those whose cInfo was not 0
 * coarse_lambda: the damping at which the current k_pcg5 coarse matrix was assembled (the inverse is reused across solves; 0 if
 * there is none).  Either pointer may be NULL. */
#define CUBA_PCG_INFO_LEN 16
#define CUBA_PCG_KERNEL_NONE 0            /* no PCG: pose-only or landmark-only systems */
#define CUBA_PCG_KERNEL_PCG 1             /* the retired first-generation k_pcg: never reported, the number stays taken */
#define CUBA_PCG_KERNEL_PCG2 2
#define CUBA_PCG_KERNEL_PCG3 3
#define CUBA_PCG_KERNEL_PCG4 4
#define CUBA_PCG_KERNEL_PCG5 5            /* k_pcg5<T, false>: the legacy shape */
#define CUBA_PCG_KERNEL_PCG5_BIG 6        /* k_pcg5<T, true> */
#define CUBA_PCG_KERNEL_PCG5T 7           /* k_pcg5t<T, K>, K = info[2] */
#define CUBA_PCG_KERNEL_DENSE 8           /* dchol::k_dense_chol: the direct solver (plan fields 0, status 0 or 2, iterations 0) */
#define CUBA_COARSE_KERNEL_NONE 0
#define CUBA_COARSE_KERNEL_INVERT 1       /* k_coarse_invert: one CTA, A <= 37 */
#define CUBA_COARSE_KERNEL_CLUSTER8 2     /* the retired k_coarse_chol_cluster2<8>: never reported, the number stays taken */
#define CUBA_COARSE_KERNEL_CLUSTER16 3    /* the retired k_coarse_chol_cluster2<16>: never reported, the number stays taken */
#define CUBA_COARSE_KERNEL_DENSE 4        /* cdense::k_coarse_dense: the whole chip, A > 37 */
#define CUBA_COARSE_KERNEL_PCG4_CLUSTER 5 /* the retired k_coarse_chol_cluster of k_pcg4: never reported, the number stays taken */
int cuba_debug_get_pcg_info(cuba_engine* e, int32_t* info, double* coarse_lambda);
/* The coarse level of k_pcg5 as the last two-level solve applied it: aggRow[numP] the aggregate of every free pose, AcP the packed
 * lower block triangle of Ac = Z^T S Z (block (ib >= jb) at (ib (ib+1)/2 + jb) * 36, column-major 6x6; 36 A (A+1)/2 doubles) and
 * AcInv its fp32 inverse [6A][6A].  Fails when no coarse level has been built.  Any pointer may be NULL. */
int cuba_debug_get_coarse(cuba_engine* e, int32_t* aggRow, double* AcP, float* AcInv);
/* Runs the dense coarse inverse k_coarse_dense, as a two-level solve launches it, on the caller's packed lower block triangle
 * AcP (layout of cuba_debug_get_coarse, A >= 1 aggregates) in buffers of its own: AcInv [6A][6A] fp32 and info 0 (inverted) or 1
 * (not positive definite: AcInv all zeros).  Needs a GPU, not a problem; no engine state changes. */
int cuba_debug_coarse_inverse(cuba_engine* e, const double* AcP, int A, float* AcInv, int* info);
/* Runs the direct solver's kernel k_dense_chol (fp64) on the caller's n x n matrix S (row-major; its lower triangle is read) and b [n],
 * in buffers of its own: x [n] and info 0 (solved) or 1 (not positive definite: x all zeros).  1 <= n <= 16380.  Needs a GPU, not a
 * problem; no engine state changes. */
int cuba_debug_dense_solve(cuba_engine* e, const double* S, const double* b, int n, double* x, int* info);
/* The two kernels of a landmark-sharded run that exchange through peer memory, with `world` ranks (1..8) emulated on this GPU:
 * the boards of every rank live in this device's memory and ONE cooperative launch runs all ranks, CTA b acting as CTA b % G of
 * rank b / G.  Both use buffers of their own and change no engine state; both fail with CUBA_ERR_INVALID when the world * G CTAs
 * cannot all be resident at once.  A rank here has numSMs / world CTAs, where a W-GPU run gives every rank the whole GPU.
 *
 * cuba_debug_peer_allreduce: `calls` consecutive all-reduces (k_peer_allreduce, G = numSMs / world, consecutive epochs on the same
 * buffers and signal blocks).  Before call c every rank's buffer is loaded with parts[c][rank][0..n) in the engine's scalar type;
 * out[c][rank][0..n) is that rank's buffer after the call. */
int cuba_debug_peer_allreduce(cuba_engine* e, int world, int64_t n, int calls, const double* parts, double* out);
/* cuba_debug_pcg5_ranks: the row-distributed k_pcg5 of a `world`-rank run on the engine's current reduced system (Hsc, bsc and the
 * poses after a Schur stage, e.g. cuba_bench_stage 3 at lambda).  The plan is build_pcg5_plan's for world ranks of numSMs / world
 * CTAs, in the launch shape setup_pcg5 gives such a plan; the preparation and one coarse setup (two_level != 0) run first, then
 * `nsolves` solves on the same boards (one launch and every rank's commit each), two-level or block-Jacobi.
 *   x [nsolves][6 numP]: the solution of each solve (rows no rank wrote are NaN);  status [nsolves][world][2]: each rank's status
 *   (0 converged, 1 iteration cap, 2 breakdown, 3 exchange abandoned) and iterations;  plan [8]: G, gs, A, needMax, maxRows, rows
 *   some other rank needs (halo rows), BIG shape (0/1), info of the coarse inverse (0 inverted, 1 not positive definite);
 *   aggRow [A+1] (may be NULL): first row of every aggregate;  AcInv [6A][6A] (may be NULL): the fp32 coarse inverse the two-level
 *   solves applied (zeros for block-Jacobi).  A <= min(numP, 148). */
int cuba_debug_pcg5_ranks(cuba_engine* e, int world, int two_level, int nsolves, double* x, int32_t* status, int32_t* plan, int32_t* aggRow,
	float* AcInv);

/* Host-only (no CUDA call): builds the index structures from the (iP,iL) lists exactly as
 * cuba_engine_set_problem does and copies them out -- the not-gpu tests check them against the oracle.
 * Sizes are returned first with all array pointers NULL, then the arrays on a second call. */
int cuba_debug_build_structure_host(const cuba_problem* p, int rank, int world, cuba_sizes* sizes,
	int32_t* hplColPtr /*numL+1*/, int32_t* hplRowInd /*nhpl*/, int32_t* edge2Hpl /*E2+E3*/,
	int32_t* hscRowPtr /*numP+1*/, int32_t* hscColInd /*nblk*/,
	int32_t* fullRowPtr /*numP+1*/, int32_t* fullColInd /*nblk_full*/,
	int32_t* shard /*[4]: lmBeg, lmEnd, edges, local products*/);

/* CPU-only check of the host side of the PCG setup (row partition over nCtas persistent CTAs, need lists, pose aggregates and
 * coarse lists of the two-level PCG, csrc/cuba_structure.cpp): builds them for the problem and verifies their invariants.
 * info[9] = G, gs, A, needMax, maxRows, blkMax, maxNeedAgg, size of the coarse lists, bytes of k_pcg3's fp64 shared memory that do
 * not hold cached blocks (set_problem fails with CUBA_ERR_INVALID when they exceed the device's budget).  No device needed. */
int cuba_debug_pcg_partition(const cuba_problem* p, int nCtas, int maxAgg, int32_t* info);

/* CPU-only check of the plan of the row-distributed two-level PCG (k_pcg5; csrc/cuba_structure.cpp): rows over world x G virtual
 * CTAs, aggregates aligned with the ranks, halo masks.  info[11] = ok (0: system too small for this kernel; then all zero), G, gs,
 * A, needMax, maxRows, maxNeedAgg, number of halo rows, blkMax, and the columns of w the polled-w staging of the fp64 shared-memory
 * layout holds in the tuned (k_pcg5t) and the legacy (k_pcg5) launch shape; a CTA polls needMax of them.  No device needed. */
int cuba_debug_pcg5_plan(const cuba_problem* p, int world, int numSMs, int maxAgg, int32_t* info);
/* The same with aggsPerCta aggregates per CTA (the one-GPU tuned kernel; 1: the plan of cuba_debug_pcg5_plan).  hash (may be null):
 * FNV-1a over every array of the plan, to compare plans across builds. */
int cuba_debug_pcg5_plan_apc(const cuba_problem* p, int world, int numSMs, int maxAgg, int aggsPerCta, int32_t* info, uint64_t* hash);
/* CPU-only: the shared-memory layout the one-GPU tuned kernel (k_pcg5t, csrc/cuba_pcg5t.cuh) gets on a device with numSMs SMs and
 * smemBudget bytes of shared memory per CTA, as set_problem picks it: the largest number of aggregates per CTA <= aggsPerCtaTop whose
 * plan exists and fits.  scalarBytes: 8 (fp64 engine) or 4.  info[12] = ok (0: no such plan; then all zero), aggregates per CTA,
 * blocks cached in shared memory per CTA, blocks of the fullest CTA left to the global copy, Z^ in shared memory, total bytes, and
 * the bytes of the cached blocks, of r / s / u, of the product staging (with the polled words), of rc, of Z^ and of the slice
 * of Ac^-1.  No device needed. */
int cuba_debug_pcg5t_layout(const cuba_problem* p, int numSMs, int aggsPerCtaTop, int scalarBytes, int64_t smemBudget, int32_t* info);
/* CPU-only: the layout the direct solver gets for the problem, as set_problem builds it.  info[5] = numP, n = 6 numP, tile rows nt =
 * ceil(n / 32), lower tiles nt (nt+1) / 2, MB of fp64 tiles; map [numP (numP+1) / 2] (may be NULL): for block (i >= j) of the packed
 * lower block triangle of S (at i (i+1)/2 + j) its index in the symmetric-full BSR of cuba_debug_build_structure_host, -1 where S has
 * no block.  CUBA_ERR_INVALID, with the message of set_problem, beyond 2730 free poses when there are free landmarks.  No device needed. */
int cuba_debug_dense_layout(const cuba_problem* p, int32_t* info, int32_t* map);
/* The flat arrays the drop-in class (cuba::CudaBundleAdjustment, csrc/cuba_api.cpp) built in its last initialize(): what optimize()
 * hands to cuba_engine_set_problem.  `dropin` is the object's address; the pointers stay valid until the next initialize().
 * Needs no GPU (tests of the graph container: tombstones, re-added edges, fixed vertices, vertices without edges). */
int cuba_debug_dropin_problem(void* dropin, cuba_problem* out);
/* The flat edge levels of the drop-in class (include/cuba_b200_levels.h), one byte per edge in the order of
 * cuba_debug_dropin_problem, with the levels set since the last initialize() applied.  The pointer stays valid until the next call
 * on the object.  Needs no GPU unless classifyEdges() ran since. */
int cuba_debug_dropin_levels(void* dropin, const uint8_t** levels, int32_t* n);

/* ---- micro-benchmark hooks for bench.py / profiles (device-resident data, CUDA-event timed) ---- */
/* Runs the named stage `reps` times back to back and returns the average device milliseconds per
 * repetition.  stage: 0 linearize (landmark pass + pose pass), 1 landmark pass only, 2 pose pass only,
 * 3 schur, 4 the reduced-system solve (PCG or dense Cholesky, as chosen), 5 backsub+update+residual, 6 residual only.  flush_l2 != 0 writes a >L2 buffer
 * between repetitions (outside the timed interval). */
int cuba_bench_stage(cuba_engine* e, int stage, int reps, int flush_l2, double lambda, double* avg_ms);

#ifdef __cplusplus
}
#endif
#endif /* CUBA_B200_H */
