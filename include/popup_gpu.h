/*
 * popup_gpu.h -- C-ABI of libpopup_gpu.so, the H100-native plane-SLAM back end.
 *
 * This is the drop-in boundary for the ONE hot path of shichaoy/pop_up_slam that this
 * repository accelerates: the factor-graph optimiser that pop_planar_slam/src/Mapping.cpp
 * drives through iSAM's C++ class API, plus the per-frame pop-up wall fit.  The reference
 * boundary is an in-process C++ API (no FFI exists upstream); every entry point below names
 * the reference interface it replaces (paths relative to the reference checkout;
 * ISAM = pop_planar_slam/Thirdparty/isam, PPS = pop_planar_slam, PUW = pop_up_wall).
 * include/isam_facade.hpp rebuilds the isam:: classes on top of this ABI so Mapping.cpp
 * compiles unchanged; INTEGRATION.md shows the binding a maintainer would add.
 *
 * Conventions
 *   - opaque handle, single-threaded per handle (the reference is single-threaded);
 *   - every function returns an int status: >= 0 success (ids / counts where documented),
 *     < 0 error, message via pus_last_error();
 *   - all arrays are caller-owned host memory, copied during the call;
 *   - node / factor ids are assigned in insertion order, per handle, starting at 0
 *     (ISAM/isamlib/Slam.cpp:47-48, Node.h:62-64, Factor.h:92);
 *   - a pose value is 7 doubles  x y z qw qx qy qz   (Pose3d = Point3d + Rot3d quaternion,
 *     ISAM/include/isam/Pose3d.h:78-79, Rot3d.h:144);
 *   - a pose measurement is 6 doubles  x y z yaw pitch roll  (Pose3d::vector(), Pose3d.h:138-145);
 *   - a plane is 4 doubles  a b c d , normalised to unit 4-norm on entry
 *     (Plane3d(const Vector4d&), PPS/src/isam_plane3d.h:59-66);
 *   - sqrt-information matrices are upper triangular, packed row-major
 *     (6 doubles for 3x3, 21 for 6x6; Noise.h:36-62, Factor.h:84-91,148-155).
 *   There is NO CPU fallback: if no CUDA device / kernel image is usable, calls fail.
 *
 * Limits (a solve fails with a message instead of producing a wrong answer):
 *   - Slam::update() only with mod_batch = 1 (what PPS sets); relative-parameterised plane factors, anchor nodes and
 *     dog-leg are not provided.  Covariances (pus_marginal_covariances, pus_covariance_blocks) are recovered only from the
 *     band solver in nested-dissection order, undamped at the estimate, within the same 8 GiB budget.
 *   - the dense direct linear solver (pus_set_linear_solver(h, 1)) handles at most 640 live poses (a dense reduced system
 *     of order 3 840, about 65 MB of device memory); a larger graph fails at upload with a message and launches nothing.
 *     The band direct solver (kind 2) takes any graph whose envelope fits 8 GiB of device memory (tiles, snapshots, pivot
 *     inverses, vectors and tables), in insertion order by default or, with pus_set_direct_ordering(h, 1), whose
 *     nested-dissection tile pattern fits the same budget; a larger one fails at upload with a message
 *     stating the need and launches nothing.  Neither spans ranks: the pus_span_* entry points refuse a direct-mode handle.
 *   - the error / Jacobian export (pus_weighted_errors .. pus_local_chi2) evaluates at the estimate only (iSAM's default
 *     Selector ESTIMATE; LINPOINT is not provided) and writes caller-owned host arrays only.  Its indices are int32: a
 *     graph whose Jacobian has more than 2^31 - 1 nonzeros is refused with a message.
 *   - the plane map (pus_map_*) covers Mapper_mono's path without loop closure (loopclose_merge, ORB bag of words); a
 *     caller's own merge removes plane nodes with pus_remove_node.  The map owns its handle's resident refresh tables.
 */
#ifndef POPUP_GPU_H
#define POPUP_GPU_H

#ifdef __cplusplus
extern "C" {
#endif

typedef void* pus_handle;

/* isam::Properties (ISAM/include/isam/Properties.h:37-110) -- the fields PPS touches
 * (PPS/src/Mapping.cpp:32-43) plus the LM constants. */
typedef struct pus_properties {
  int method;              /* 0 GAUSS_NEWTON (default), 1 LEVENBERG_MARQUARDT */
  double epsilon2;         /* stop when ||delta|| <= epsilon2        (1e-2) */
  double epsilon_abs;      /* stop when chi2 <= epsilon_abs          (1e-3) */
  double epsilon_rel;      /* stop when d(chi2) < epsilon_rel*chi2   (1e-5) */
  int max_iterations;      /* (500) */
  double lm_lambda0;       /* (1e-6) */
  double lm_lambda_factor; /* (10) */
  int mod_update;          /* (1) */
  int mod_batch;           /* (100); PPS sets 1 */
  int mod_solve;           /* (1) */
} pus_properties;

/* Solver knobs that have no counterpart in the reference (it uses a direct CHOLMOD solve,
 * ISAM/isamlib/Cholesky.cpp:68-147; here the reduced pose system is solved by block-PCG). */
typedef struct pus_solver_options {
  double pcg_rel_tol;  /* ||r||_Minv / ||b||_Minv target, default 1e-8 (four decades under the 1e-4 parity bar).  At 1e-7 the bench
                        * workload is 8 % faster and still follows the reference trajectory, but the estimates of an UNCONVERGED
                        * 4 200-pose Huber corridor after 5 capped iterations drift to 1.15e-4 of the oracle's: too close to the bar */
  int pcg_max_iter;    /* default 2000 */
  int ctas_per_sm;     /* persistent grid = ctas_per_sm * #SM, 0 = auto */
  int team_ctas;       /* CTAs cooperating on one graph; 0 = auto (whole grid for one graph) */
  int reserved[4];     /* diagnostics, all 0 by default:
                        *   [0] = 1  rebuild the preconditioner for every linear solve (no lazy refresh)
                        *   [1] = 1  no PCG warm start after a rejected LM step
                        *   [2]      bit 0: sub-phase timers in pus_stats.phase_ms[13..23]; bit 1: always stage W / Wt
                        *            tiles by bulk async copy (the large-graph data path); bit 2: never; bit 3: force the
                        *            three-level preconditioner (default: graphs > 5120 poses); bit 4: force two levels;
                        *            bit 5: no block-resident PCG loop; bit 6: another timer set; bits 8-15: the CTA of the
                        *            team that keeps the timers; bit 16: never run a team as a thread-block cluster (global-
                        *            memory barrier only; the environment variable PUS_CLUSTER=0 does the same process-wide)
                        *   [3] > 0  lazy-refresh threshold in percent of the post-build iteration count (default 130, three
                        *            levels 200) */
} pus_solver_options;

typedef struct pus_stats {
  int lm_iterations;      /* trial steps of the last batch_optimize (Optimizer.cpp num_iter) */
  int accepted;           /* accepted steps */
  int relinearizations;   /* Jacobian sweeps */
  int chi2_evals;         /* trial chi2 sweeps */
  long long pcg_iterations; /* total PCG iterations of the last call */
  double chi2_initial, chi2_final;
  double kernel_ms;       /* device time of the solve kernel(s), CUDA events on the handle's stream */
  double h2d_ms, d2h_ms;
  long long h2d_bytes, d2h_bytes;
  int n_poses, n_planes, n_pose_plane, n_odometry, n_pose_prior, n_plane_prior;
  int gpu_launches;       /* kernels launched by the last call */
  int grid_ctas, block_threads;
  double phase_ms[24];    /* in-kernel %globaltimer split: 0 linearise, 1 Schur set-up, 2 PCG, 3 back-substitution + update,
                             4 chi2; 8..12 set-up parts (Hll^-1, dense blocks, Wc, A_c, A_c^-1); 16..20 PCG parts
                             (plane sweep, plane solve, pose sweep, pose side + dot, preconditioner + dot) */
} pus_stats;

/* ---- lifetime ------------------------------------------------------------------------- */
/* isam::Slam::Slam()  ISAM/isamlib/Slam.cpp:69-78 */
int pus_create(int device, pus_handle* out);
int pus_destroy(pus_handle h);
const char* pus_last_error(void);
/* run the solve kernels on this CUDA stream (cudaStream_t as void*), 0 = library-owned stream */
int pus_set_stream(pus_handle h, void* cuda_stream);

/* ---- vertices --------------------------------------------------------------------------- */
/* new Pose3d_Node() + Slam::add_node  (slam3d.h:39, Slam.cpp:91-94; PPS Mapping.cpp:464-465).
 * init7 may be NULL (uninitialised node, NodeT::NodeT Node.h:107-110). Returns the node id. */
int pus_add_pose(pus_handle h, const double* init7);
/* new Plane3d_Node() + add_node  (isam_plane3d.h:197-210; Mapping.cpp:483-484) */
int pus_add_plane(pus_handle h, const double* abcd);
/* bulk forms: values may be NULL; out_ids may be NULL; returns the first id */
int pus_add_poses(pus_handle h, int n, const double* init7s, int* out_ids);
int pus_add_planes(pus_handle h, int n, const double* abcds, int* out_ids);
/* NodeT::init  Node.h:123-126 (Mapping.cpp:475, 499) */
int pus_init_pose(pus_handle h, int id, const double* init7);
int pus_init_plane(pus_handle h, int id, const double* abcd);
/* bulk NodeT::init over n vertices (values packed like the single-vertex forms) */
int pus_init_poses(pus_handle h, int n, const int* ids, const double* init7s);
int pus_init_planes(pus_handle h, int n, const int* ids, const double* abcds);
/* NodeT::value()  Node.h:130 */
int pus_get_pose(pus_handle h, int id, double* out7);
int pus_get_plane(pus_handle h, int id, double* out4);
int pus_get_poses(pus_handle h, int n, const int* ids, double* out7s);
int pus_get_planes(pus_handle h, int n, const int* ids, double* out4s);

/* ---- edges ------------------------------------------------------------------------------ */
/* Pose3d_Factor(node, prior, noise) + add_factor  (slam3d.h:58-89; Mapping.cpp:472-473) */
int pus_add_pose_prior(pus_handle h, int pose, const double* xyzypr, const double* sqrtinf_ut21);
/* Pose3d_Pose3d_Factor(n1, n2, measure, noise) + add_factor  (slam3d.h:91-193; Mapping.cpp:477-478).
 * Initialises whichever pose is uninitialised (slam3d.h:123-137). */
int pus_add_odometry(pus_handle h, int pose1, int pose2, const double* xyzypr, const double* sqrtinf_ut21);
/* Pose3d_Plane3d_Factor(pose, plane, measure, noise, relative=false) + add_factor
 * (isam_plane3d.h:221-308; Mapping.cpp:513,523). Initialises the plane on first sight (:252-264). */
int pus_add_pose_plane(pus_handle h, int pose, int plane, const double* meas_abcd, const double* sqrtinf_ut6);
/* Plane3d_Factor(plane, prior, noise) + add_factor  (isam_plane3d.h:428-474; Mapping.cpp:502-503) */
/* Pose3d_Plane3d_Factor2 (pop_planar_slam/src/isam_plane3d.h:314-424): like pus_add_pose_plane, but the residual
 * re-pops the measured wall plane from the two precomputed ground-edge rays (sensor frame, rays6 = r0, r1 as
 * precompute_edge_ray :358-370 forms them: invK * (x, y, 1)) with the CURRENT pose on every evaluation
 * (get_wall_plane_equation, isam_plane3d.cpp:20-55); meas4 only initialises an un-initialised plane node. */
int pus_add_pose_plane2(pus_handle h, int pose, int plane, const double* meas4, const double* rays6, const double* sqrtinf_ut6);
int pus_add_plane_prior(pus_handle h, int plane, const double* abcd, const double* sqrtinf_ut6);
/* bulk forms (same semantics, applied in array order); out_fids may be NULL; returns first fid */
int pus_add_odometry_bulk(pus_handle h, int n, const int* pose1, const int* pose2, const double* xyzypr,
                          const double* sqrtinf_ut21, int* out_fids);
int pus_add_pose_plane_bulk(pus_handle h, int n, const int* pose, const int* plane, const double* meas_abcd,
                            const double* sqrtinf_ut6, int* out_fids);
/* FactorT::set_measurement / measurement()  Factor.h:203-206 (Mapping.cpp:603, 668) */
int pus_set_measurement(pus_handle h, int fid, const double* meas);
int pus_get_measurement(pus_handle h, int fid, double* meas);
/* Slam::remove_factor / remove_node  Slam.cpp:107-126 (Mapping.cpp:673, 699) */
int pus_remove_factor(pus_handle h, int fid);
int pus_remove_node(pus_handle h, int id);
/* Graph::num_nodes / num_factors  Graph.h:61-62 (Mapping.cpp:547-548) */
int pus_num_nodes(pus_handle h);
int pus_num_factors(pus_handle h);
/* Factor::nodes() Factor.h:79 / Node::factors() Node.h:88 (Mapping.cpp:664, 667) */
int pus_factor_nodes(pus_handle h, int fid, int* out2);             /* returns #nodes */
int pus_node_factors(pus_handle h, int id, int* out, int capacity); /* returns #factors (insertion order) */
/* column offset of a node / row offset of a factor in the stacked Jacobian
 * (Slam::update_starts Slam.cpp:59-67; jacobian_partial Slam.cpp:395-432) -- the
 * "edge indexing bit-exact" contract. -1 if removed. */
int pus_node_start(pus_handle h, int id);
int pus_factor_row(pus_handle h, int fid);

/* ---- configuration ---------------------------------------------------------------------- */
/* Slam::properties / set_properties  Slam.h:92-101 (Mapping.cpp:32-43) */
int pus_get_properties(pus_handle h, pus_properties* out);
int pus_set_properties(pus_handle h, const pus_properties* in);
/* Slam::set_cost_function  Slam.cpp:212-214 with robust.h:101-118:
 * kind 0 none, 1 cost_huber(d,b), 2 cost_pseudo_huber(d,b); applied per residual component
 * (Factor.h:67-77). */
int pus_set_robust(pus_handle h, int kind, double b);
/* Properties::force_numerical_jacobian (ISAM/include/isam/Properties.h:44-45) / Factor::jacobian -> numericalDiff
 * (Factor.h:126-139, ISAM/isamlib/numericalDiff.cpp:41-87).  numeric = 0 (default): closed-form Jacobian blocks;
 * numeric = 1: the reference's own scheme on the device -- central differences, epsilon = 1e-4, through the exmaps, of the
 * weighted robustified residual, linearisation point restored through the Euler round trip as upstream.  With it a solve
 * follows the reference's trajectory (same accept / reject sequence) where its truncation error decides near-tie steps. */
int pus_set_jacobian_mode(pus_handle h, int numeric);
/* Linear solver of the reduced pose system S dp = b (DESIGN.md section 5); a handle setting, no iSAM counterpart.
 * kind 0 (default): block-preconditioned CG to pcg_rel_tol.  kind 1: exact -- S assembled densely on the device, factored
 * S = L L^T (48x48 tiles, FP64 tensor cores) and solved by two blocked triangular solves, as the reference's direct
 * Cholesky (ISAM/isamlib/Cholesky.cpp:68-147) solves the same damped system.  kind 2: exact as kind 1, on the envelope of
 * a bordered system -- the poses in insertion order, then the few planes seen from most of the trajectory (chosen by
 * observer span, at most 64) kept as unknowns instead of being eliminated; the tiles outside the envelope are never stored,
 * factored or read (DESIGN.md section 5.2); pus_set_direct_ordering picks the order of kind 2's pose tiles.  Every linear solve is bit-identical across
 * team sizes, barrier kinds and batch positions; the chi2 and |delta| of the trace come from the team reduction, whose order
 * follows the team size, so whole runs agree bit for bit as long as no accept / reject decision is a tie in the last bits.  It applies to pus_batch_optimize (LM and GN), pus_update, pus_solve_resident
 * and the _many forms; a batch may mix all kinds (PCG and direct handles run as launches of their own).  In direct mode
 * pus_get_trace's pcg entry is 0 for a step whose factorization succeeded and -1 for one that met a non-positive pivot
 * (the step is then delta = 0: LM evaluates it as a trial step, rejects it and raises lambda; GN stops; pus_update applies
 * the zero step, leaving the estimate where it was), pus_stats.pcg_iterations is 0, phase_ms[1] is
 * assembly + factorization and phase_ms[2] the triangular solves + plane back-substitution, and the set-up sub-slots are
 * 8 plane inverses, 10 (pose, plane) blocks W and W Hll^-1, 11 assembly of S, 12 factorization, 13 right-hand side,
 * 14 triangular solves.  Limits: see the header's Limits block.  Changing the kind lays the graph out again at the next
 * upload.  The debug hooks of direct mode ("Sdir", "Ldir", stages 4 and 5) use the bordered order in kind 2: 6 N pose rows,
 * then 3 per bordered plane; a stored "Sdir" must lie inside the envelope, and stage 5 writes the bordered planes' part of
 * the solution to their dl. */
int pus_set_linear_solver(pus_handle h, int kind);
int pus_get_linear_solver(pus_handle h);   /* the kind, or < 0 on error */
/* Order of the band solve's pose tiles (kind 2 only; a handle setting, accepted at any time).  order 0 (default): insertion
 * order, the envelope layout.  order 1: nested dissection -- the 8-pose tiles permuted by recursive bisection of the tile
 * graph (separators last, the bordered planes chosen by the number of pose tiles that see them and ordered after every
 * pose), stored as L's tile pattern and factored level by level of the elimination tree (DESIGN.md section 5.3).  It keeps
 * the fill near linear where insertion order has a wide envelope, as on a map whose loop closure re-observes earlier
 * planes.  Other values are refused.  Changing it lays the graph out again at the next upload.  Debug hooks in order 1:
 * "Sdir" and stages 4 / 5 keep the bordered order (a stored "Sdir" must lie inside the pattern), "Ldir" is the factor of
 * P S P^T in the permuted order; "ndtile" (new column -> original tile), "ndparent", "ndcptr" / "ndcrow" (L's pattern per
 * column), "ndlevel", "ndtoff" / "ndtrow" / "ndtcol" (tile storage) and "nduptr" / "ndupd" (update lists) fetch the tables. */
int pus_set_direct_ordering(pus_handle h, int order);
int pus_get_direct_ordering(pus_handle h);   /* the order, or < 0 on error */
int pus_get_solver_options(pus_handle h, pus_solver_options* out);
int pus_set_solver_options(pus_handle h, const pus_solver_options* in);

/* ---- optimisation ----------------------------------------------------------------------- */
/* int Slam::batch_optimization()  Slam.cpp:198-210 -> Optimizer::batch_optimize
 * (Optimizer.cpp:538-555): GN (286-366) or LM (371-467) per properties.method.
 * Host graph -> HBM, device-resident loop, estimates -> host mirrors. */
int pus_batch_optimize(pus_handle h, int* iterations);
/* UpdateStats Slam::update()  Slam.cpp:157-196; with mod_batch==1 (PPS) = relinearise +
 * one un-damped Gauss-Newton step (Optimizer::relinearize Optimizer.cpp:114-185). */
int pus_update(pus_handle h);
/* double Slam::chi2()  Slam.cpp:266-268 (ESTIMATE) */
int pus_chi2(pus_handle h, double* out);
/* many independent graphs in one launch (BASELINE config 4); one CTA team per graph.
 * Every *_many call (here, the split calls below and pus_span_emulate_optimize) takes an array of n distinct, non-null
 * handles: a null array, a null entry or a handle listed twice is refused with a message before any device work (two
 * teams would otherwise solve one graph's device buffers at once).  n <= 0 does nothing and returns 0.  The handles ride
 * on the first handle's stream for the duration of the call and get their own streams back when it returns. */
int pus_batch_optimize_many(pus_handle* hs, int n, int* iterations);

/* split form of pus_batch_optimize for measurement: upload (graph compile + H2D),
 * solve from the uploaded initial estimate with everything resident in HBM (repeatable),
 * download (D2H into the host mirrors).
 * The resident solve and the download act on the graph as it was uploaded: a structural edit (node or factor added or
 * removed), a change of linear-solver kind or of direct ordering after pus_upload makes them refuse the handle with
 * "graph changed since its upload: call pus_upload", and nothing is launched or copied.  Value and measurement changes
 * (pus_init_*, pus_set_measurement) do not make a handle stale: the resident solve starts again from the uploaded
 * estimate and measurements, and pus_download overwrites the host values with its result; pus_upload takes them in.
 * pus_batch_optimize and pus_batch_optimize_many upload first and are not affected. */
int pus_upload(pus_handle h);
int pus_solve_resident(pus_handle h, int* iterations);
int pus_download(pus_handle h);
int pus_upload_many(pus_handle* hs, int n);
int pus_solve_resident_many(pus_handle* hs, int n, int* iterations);
int pus_download_many(pus_handle* hs, int n);

int pus_get_stats(pus_handle h, pus_stats* out);
/* per LM trial step: lambda used, chi2 of the trial, chi2 before, ||delta||, accepted flag,
 * PCG iterations of the solve that produced delta. Returns the number of entries. */
int pus_get_trace(pus_handle h, int capacity, double* lambda, double* chi2_new, double* chi2_before,
                  double* delta_norm, int* accepted, int* pcg_iters);

/* ---- pop-up wall fit (float32) ---------------------------------------------------------- */
/* popup_plane::get_plane_equation (PUW/libs/popup_plane.cpp:551-652, mode 0, also
 * update_plane_equation_from_seg :654-705) and update_plane_equation_from_seg_fast
 * (:708-749, mode 1), batched over frames:
 *   seg_ptr[n_frames+1]  CSR offsets into segs (4 floats each: x1 y1 x2 y2, pixels)
 *   invK[9] row-major, Ts[n_frames*16] row-major camera-to-world
 *   outputs have one row per (frame, plane) with plane 0 = ground, i.e. n_seg(f)+1 rows
 *   per frame at row offset seg_ptr[f]+f:  planes_world/sensor 4 floats, dist 1, good 1 (0/1).
 * A seg_ptr that is NULL, does not start at 0 or decreases is refused before any device work.
 * Any output may be NULL. */
int pus_popup_fit_frames(int device, int n_frames, const int* seg_ptr, const float* segs, const float* invK,
                         const float* Ts, float dist_thre, int mode, float* planes_world, float* planes_sensor,
                         float* dist, int* good);

/* ---- dense plane clouds (float32) ------------------------------------------------------------------ */
/* popup_plane::generate_cloud (PUW/libs/popup_plane.cpp:807-863) with closed_polygons_homo_pts (:81-116) and
 * matrixToCloud (:925-985), batched over frames and their good planes, on the device:
 *   plane_ptr[n_frames+1]   CSR offsets of the frames' planes, in the caller's order; the first plane of every frame is the
 *                           ground (label 255), the others walls (label 0), as in pus_popup_fit_frames' rows
 *   poly_ptr[n_planes+1], polys[n_vertices][2]   each plane's closed 2-D polygon (float pixels); an empty one gives no points
 *   planes_sensor[n_planes][4]   the plane in the sensor frame (pus_popup_fit_frames' planes_sensor rows)
 *   Ts[n_frames][16] row-major camera-to-world, invK[9] row-major
 *   images[n_frames][height][width][3]   packed BGR, or NULL (colour 0, no border rule); width and height are needed either way
 *   downsample   halve the polygon, fill, double the pixel coordinates (generate_cloud's downsample_poly)
 * Per pixel: the polygon (halved when downsampling) is truncated to integer points, filled on its bounding box with
 * cv::fillConvexPoly's rule (OpenCV 4.13, LINE_8, shift 0; non-convex, degenerate and partly off-image polygons included) and
 * listed in cv::findNonZero order.  ray = invK (x, y, 1), p_s = -d / (n . ray) ray (ray_plane_interact), p_w = R p_s + t.
 * Points with p_s.z < 0, p_s.z > depth_thre or p_w.z < -0.2 are dropped, z is clamped to ceiling_threshold, and with
 * 960-wide images pixels with x < 4 or y < 4 are dropped.
 * Outputs (any may be NULL): counts[n_planes] kept points per plane, offsets[n_planes] their first index; xyz[total][3] and
 * rgb[total][3] (r, g, b) the per-plane clouds back to back, which is also the frame's mixed cloud; capacity is their room in
 * points (xyz = rgb = NULL is a size query, too small a capacity fails with a message); labels[n_frames][height][width]
 * 127 void / 255 ground / 0 wall, with the nearest-neighbour 0.5x / 2x resize in downsample mode (even sizes only).
 * Returns the total number of points.  The outputs are deterministic: repeated calls and any split of the batch give the
 * same bytes.  Two deviations from the reference, where it is undefined: pixels outside the image keep their points with
 * colour 0 and are not written to the label image (the reference reads and writes out of bounds), and a call without images
 * gives colour 0 (the reference keeps the previous point's colour).  The fill is pinned to OpenCV 4.13; differences of older
 * OpenCV releases are not reproduced.  Polygons have at most PUS_POPUP_MAX_VERTICES vertices and coordinates of magnitude
 * at most PUS_POPUP_MAX_COORD. */
#define PUS_POPUP_MAX_VERTICES 256
#define PUS_POPUP_MAX_COORD 1048576.0f
long long pus_popup_clouds(int device, int n_frames, const int* plane_ptr, const int* poly_ptr, const float* polys,
                           const float* planes_sensor, const float* Ts, const float* invK, const unsigned char* images,
                           int width, int height, int downsample, float depth_thre, float ceiling_threshold, int* counts,
                           long long* offsets, float* xyz, unsigned char* rgb, long long capacity, unsigned char* labels);

/* ---- closed wall and ground polygons (float32) ------------------------------------------------------------------ */
/* popup_plane::find_2d_3d_closed_polygon (PUW/libs/popup_plane.cpp:120-406, simple_polygon_mode = false) with
 * direction_hit_boundary and cut_wall_polygons (PUW/libs/matrix_utils.cpp:229-270, 506-713), batched over frames, on the
 * device.  The step between get_plane_equation (pus_popup_fit_frames) and generate_cloud (pus_popup_clouds):
 *   seg_ptr[n_frames+1], segs   the frames' connected ground segments, as pus_popup_fit_frames
 *   K[9], invK[9] row-major, Ts[n_frames][16] row-major camera-to-world; width, height the image size
 *   ceiling_threshold   the cut height; walllength_threshold   the cut length from the ground endpoint nearer the camera
 *                       (negative: height only, as cut_wall_polygons tests it)
 * Rows as pus_popup_fit_frames': n_seg(f) + 1 per frame at seg_ptr[f] + f, row 0 the ground.  Per row:
 *   bound2d   the closed 2-D polygon out to the image border (all_closed_2d_bound_polygons)
 *   world3d   a wall's polygon on its plane in the world frame, cut (all_3d_bound_polygons_world); empty for the ground,
 *             which the reference never assigns
 *   cut2d     world3d projected back through K (all_closed_2d_cutted_polygons); the ground's is its bound polygon
 * Counts per row ([n_rows] each) are always written; the vertices are packed in row order (2 or 3 floats each), so both
 * 2-D sets are the poly_ptr / polys input of pus_popup_clouds.  bound2d = cut2d = world3d = NULL is a size query; the
 * capacities are in vertices, and too small a one fails with a message.  Frames without segments give empty rows.
 * The planes and world ground endpoints come from the same device code as pus_popup_fit_frames (mode 0).  The cut follows
 * OpenCV 4.13's cv::convexHull (start vertex, orientation, dropped collinear and duplicate points) and cv::pointPolygonTest
 * on Point2f; point sets with three points collinear only up to float rounding are outside that guarantee (OpenCV's
 * result there depends on how its build contracts the orientation test).  Deviations: the camera inverse is
 * [R^T | -R^T t] in closed form (Eigen's general inverse may differ in the last bit); float -> int truncations follow x86
 * (NaN or out of range gives INT_MIN); where find_correct_ground_seq would index past its hull the uncut polygon is kept,
 * as when it finds no sequence; nothing is printed.  Deterministic: repeated calls and any split of the batch give the
 * same bytes.  There is no CPU fallback. */
#define PUS_POPUP_MAX_SEGMENTS (PUS_POPUP_MAX_VERTICES - 6)   /* a ground polygon has n + 6 vertices at most */
int pus_popup_polygons(int device, int n_frames, const int* seg_ptr, const float* segs, const float* K, const float* invK,
                       const float* Ts, int width, int height, float ceiling_threshold, float walllength_threshold,
                       int* bound_counts, int* cut_counts, int* world_counts, float* bound2d, float* cut2d, float* world3d,
                       long long bound_capacity, long long cut_capacity, long long world_capacity);

/* ---- pop-up depth map (float32) ------------------------------------------------------------------ */
/* popup_plane::get_depth_map_good (PUW/libs/popup_plane.cpp:866-921), the depth init of the popped-up scene, batched over
 * frames, on the device.  The inputs mean what they mean for pus_popup_clouds: plane_ptr[n_frames+1] the frames' good planes
 * in order, poly_ptr / polys each plane's closed 2-D bound polygon (pus_popup_polygons' bound2d rows), planes_sensor their
 * sensor-frame planes (pus_popup_fit_frames' planes_sensor rows), Ts camera-to-world, invK, the image size and downsample.
 * Per frame the map starts at 0 and its planes are drawn in order, a later plane over an earlier one.  Each polygon's pixels
 * are those of pus_popup_clouds (OpenCV 4.13's fillConvexPoly + findNonZero, halved and doubled in downsample mode).  Per
 * pixel, ray = invK (x, y, 1), p_s = -d / (n . ray) ray, p_w = R p_s + t:
 *   p_w.z < ceiling_threshold   write p_s.z, unless p_s.z < 0 (the pixel keeps its earlier value)
 *   otherwise                   write the z of ray's hit on the ceiling plane T^T (0, 0, -1, ceiling_threshold), unless it
 *                               is < 0
 * The comparisons are the reference's: a NaN height takes the ceiling branch and a NaN depth under a finite height is written.
 * With downsample the map of a frame with planes is then resized as the reference does: cv::resize 0.5x (INTER_LINEAR, which
 * OpenCV runs as its area fast path at 0.5), convertTo x4, cv::resize 2x INTER_LINEAR, bit for bit as OpenCV 4.13's own code;
 * width and height must then be even (the reference's round trip changes the size of an odd image).
 * depth[n_frames][height][width] receives the maps.  Deterministic, no floating-point atomics: repeated calls and any split
 * of the batch give the same bytes.  Refusals (malformed CSR offsets, more than PUS_POPUP_MAX_VERTICES vertices, a
 * coordinate not finite or beyond PUS_POPUP_MAX_COORD, a non-positive size, odd sizes in downsample mode, no depth) fail with
 * a message and launch nothing; there is no CPU fallback.  Deviations from the reference:
 *   - pixels outside the image are not written (the reference writes out of bounds);
 *   - a plane is skipped when the polygon passed in is empty (the reference tests its member all_closed_2d_bound_polygons but
 *     fills from the argument);
 *   - the ceiling plane is always formed from Ts and ceiling_threshold (the reference takes it as an argument);
 *   - the resize follows OpenCV's own code, not the Intel IPP build that the pip wheels enable by default, whose 2x
 *     INTER_LINEAR differs by up to 3 ulp. */
int pus_popup_depth(int device, int n_frames, const int* plane_ptr, const int* poly_ptr, const float* polys,
                    const float* planes_sensor, const float* Ts, const float* invK, int width, int height, int downsample,
                    float ceiling_threshold, float* depth);

/* ---- ground edges (float32) ------------------------------------------------------------------ */
/* popup_plane::edge_get_polygons (PUW/libs/select_edge.cpp:66-406) with the Python stages it runs through an embedded
 * interpreter, pop_up_fun.python_get_contours and interval_tree_optimization (pop_up_python/python/pop_up_python/
 * pop_up_fun.py:85-205), batched over frames, on the device: which of a frame's detected lines form the ground-wall
 * boundary, given the CNN label map.  The lines come from pus_popup_lines (below) or the caller's own detector.
 * PUS_POPUP_MAX_LINES stays this call's limit even though pus_popup_lines may give a frame more lines.
 *   labels[n_frames][height][width]   the label maps, ground 255 (any uint8 values are taken)
 *   line_ptr[n_frames+1], lines[n][4]   CSR offsets and the frames' detected lines x1 y1 x2 y2 (float pixels)
 *   params   popup_plane's members (popup_plane.h:178-200); NULL is refused
 * Outputs, as edge_get_polygons' return tuple, packed in frame order like pus_popup_polygons':
 *   open_counts[n_frames], open_segs[..][4]        ground_seg2d_lines_actual, what main_3d.cpp:428 passes to the fit: the
 *                                                  counts prefix-summed are pus_popup_fit_frames' seg_ptr, open_segs its segs
 *   connect_counts[n_frames], connect_segs[..][4]  ground_seg2d_lines_connect: the same segments with the connectors added
 *   open_in_connect[..]                            final_lines_in_extend_ind: each open segment's row in its frame's
 *                                                  connected list
 *   status[n_frames]   0 segments found; 1 no contour (the Python raises; the reference then reads a missing or stale
 *                      ground_contour), also when the assembly would raise KeyError (a dict pop of a key it never stored,
 *                      which scikit-image 0.14's lookups by get allow where pixels are shared by several chains);
 *                      2 nothing survives steps 1-4 (the reference returns empty lists); 3 the interval tree would raise
 *                      on a null or reversed interval; 4 no segment is longer than post_short_thre (the reference then
 *                      indexes an empty matrix); 5 the frame's scratch ran out: the contour assembly's node list (4 nodes
 *                      per marching-squares segment, of which a join through a stale dict entry may copy a contour) --
 *                      a limit of this library, not an outcome of the reference.  A frame with a non-zero status has
 *                      no segments.
 * The counts and status are always written; open_segs = connect_segs = NULL is a size query; the capacities are in rows,
 * and too small a one fails with a message.  Returns the number of frames with status 0.
 * Stages, pinned:
 *   0 labels: with downsample_contour cv::resize 0.5x INTER_NEAREST (source pixel min(2 x, w - 1); the half size rounds
 *     half to even as cvRound), dilate 8 x 8, erode 8 x 8; otherwise dilate dilation_distance^2 and erode erosion_distance^2.
 *     A k x k box with OpenCV's anchor k / 2 and its default border (pixels outside take no part), then 255 - v; OpenCV 4.13.
 *   1 contour: scikit-image 0.14's find_contours(map, 0) (cells row-major, case bits ul > 0 (1), ur (2), ll (4), lr (8),
 *     saddles 6 and 9 fully_connected='low', degenerate segments skipped, joined through its two point-keyed dicts, stale
 *     entries and the lower contour number's survival included, sorted by number); at level 0 on uint8 data every point is
 *     a pixel.  The contour with the largest start-end distance (first maximum), as (x, y), every 20th point but the last,
 *     doubled with downsample_contour.
 *   2 steps 1-4 of select_edge.cpp:91-257, each restart loop capped at 100 passes acting on the first triggering pair.
 *   3 intervaltree 2.x: a set of (begin, end, data) intervals, half-open search, sorted by (begin, end, data),
 *     split_overlaps at every boundary; overlap sums in float64 of float32 terms and the int() refinement in float64, as
 *     NumPy 1.x promotes a float32 scalar with a Python number.
 *   4 post-processing of select_edge.cpp:276-405, direction_hit_boundary as pus_popup_polygons'.
 * Precision: the thresholds are doubles and compared in double against float values; sample_ind / 10.0 rounds to float;
 * PI = 3.14159265.  Deviation: angles use float(atan2(double y, double x)) on every side instead of atan2f, whose glibc and
 * CUDA versions differ (at most 1 ulp).  Refused with a message, nothing launched: malformed line_ptr, non-finite lines,
 * more than PUS_POPUP_MAX_LINES lines in a frame, width or height below 4, NULL labels or params, kernel sizes below 1.
 * Deterministic (no floating-point atomics): repeated calls and any split of the batch give the same bytes.  No CPU
 * fallback. */
#define PUS_POPUP_MAX_LINES 512
typedef struct pus_edge_params {
  int dilation_distance, erosion_distance;   /* 11, 11 (k x k box); with downsample_contour 8 x 8 on the half map */
  int downsample_contour;                    /* popup_param.yaml: true; popup_tum_far.yaml: false */
  double pre_vertical_thre, pre_minium_len, pre_boundary_thre, pre_contour_close_thre, pre_merge_angle_thre,
      pre_merge_dist_thre, pre_proj_angle_thre, pre_proj_cover_thre, pre_proj_cover_large_thre, pre_proj_dist_thre,
      interval_overlap_thre, post_short_thre, post_bind_dist_thre, post_merge_dist_thre, post_merge_angle_thre,
      post_extend_thre;
} pus_edge_params;
int pus_popup_edges(int device, int n_frames, const unsigned char* labels, int width, int height, const int* line_ptr,
                    const float* lines, const pus_edge_params* params, int* status, int* open_counts, int* connect_counts,
                    float* open_segs, float* connect_segs, int* open_in_connect, long long open_capacity,
                    long long connect_capacity);

/* ---- line detection (float32) ------------------------------------------------------------------ */
/* The detector half of popup_plane::get_ground_edges (popup_plane.cpp:753-770): grey, contrast and
 * line_lbd_detect::detect_raw_lines with use_LSD = false (main_3d.cpp:417-424), i.e. line_lbd's EDLines
 * (binary_descriptor.cpp: detectImpl, OctaveKeyLines, EDLineDetector::EdgeDrawing / EDline) in the configuration the SLAM
 * pipeline runs: one octave, the EDLineDetector() defaults (gradient threshold 80, anchor threshold 8, scan interval 2,
 * minimum line length 15, fit error threshold 1.6, TryTime 6, SkipEdgePoint 2), an all-ones mask.  Batched over frames.
 *   images[n_frames][height][width][channels]   channels 3 (BGR, as pus_popup_clouds takes them) or 1 (grey, used as is)
 *   downsample   popup_plane's use_fast_edges_detection: detect on the 0.5x image, lines scaled by 2
 * Outputs: counts[n_frames] and status[n_frames] (always written); lines[total][4] x1 y1 x2 y2, packed in frame order,
 * so that the prefix sum of counts is pus_popup_edges' line_ptr and lines its lines as is.  lines = NULL is a size query;
 * capacity is in rows and too small a one fails with a message.  Returns the total number of lines.
 *   status 0 lines found (possibly none); 1 EdgeDrawing's arrays would overflow -- more anchors than N / 5, more edge
 *          pixels than N / 5 in either half, or more chains than N / 100 (N the detection image's pixels).  The reference
 *          writes past its arrays before it checks these limits, then prints an error, and detectImpl ignores the -1:
 *          the frame gets no lines.  Here likewise: status 1, no lines.
 * Stages, pinned (OpenCV 4.13 on 8-bit data):
 *   1 grey: cvtColor BGR2GRAY, (3735 B + 19235 G + 9798 R + 2^14) >> 15.
 *   2 contrast: if the integer pixel sum times 1.0 / N (double) is below 90, equalizeHist: LUT from the first non-empty
 *     bin i (0 there), saturate_cast<uchar>(float(cumulative count) * (255.f / (N - hist[i]))), round half to even; an
 *     image of one value maps every pixel to itself.
 *   3 downsample: resize 0.5 x INTER_LINEAR, which OpenCV runs on 8U as its area path: (a + b + c + d + 2) >> 2.  Odd
 *     sizes are refused in this mode.
 *   4 blur: GaussianBlur 5 x 5, sigma 1, the bit-exact fixed-point filter (14 62 104 62 14) / 256 per pass, rows kept
 *     with 8 fractional bits, columns rounded from 16; BORDER_REFLECT_101.
 *   5 Sobel 3 x 3 to CV_16S (BORDER_REFLECT_101), |dx| + |dy|, THRESH_TOZERO at 81, / 4 as saturate_cast<short>(v * 0.25f)
 *     (round half to even: 82 -> 20, 86 -> 22); direction Horizontal where |dx| < |dy|.
 *   6 anchors scanned column-major (x outer, y inner), both from 1 in steps of 2.
 *   7 edge drawing in anchor order: neighbour comparisons on the gradient's low byte ((unsigned char) of the short), the
 *     loop condition on the full short; the last position carried from walk to walk; the anchor unmarked between the two
 *     half-walks and its second copy skipped in the chain; chains under 16 pixels dropped with their pixels left marked.
 *   8 per chain: LeastSquaresLineFit_ (both forms: Mat_<float> matrices, products accumulated in double and rounded to
 *     float once as OpenCV's gemm, ATA + tmp a float add, the solve in double; a singular fit gives NaN, which fails every
 *     comparison), the extension with up to 3 popped-back outliers and TryTime, LineValidation_ and nfa in double,
 *     endpoints computed in double and stored as float.
 *   9 OctaveKeyLines' endpoint swap: the float direction against double multiples of M_PI (a direction that rounds to
 *     float pi lies beyond M_PI and takes no range); then keylines_to_mat's float rows (times 2 with downsample).
 * Deviations, where the reference is undefined:
 *   - the overflow cases above (status 1);
 *   - the mask test reads the all-ones mask at projected endpoints that can lie just outside the image: here no line is
 *     ever removed;
 *   - an initial fit that ends NaN at the end of a chain makes the reference read past the chain to form a line that its
 *     validation always rejects: here the chain simply ends;
 *   - EDline sizes its line index array 5 x chains and writes past it when a frame has more lines: here every line is
 *     kept.
 * The transcendentals of the validation (atan2 and nfa's log, exp, sinh, pow, log10) are CUDA's on the device and
 * glibc's on the host, which may differ by an ulp; only the decisions they feed (nfa > 0, |angle difference| <
 * 0.392699, the direction ranges) reach the output.  There is no per-frame line cap: a frame may give more than
 * PUS_POPUP_MAX_LINES lines, which pus_popup_edges refuses as before.  Refused with a message, nothing launched: NULL
 * images, status or counts, channels other than 1 or 3, odd sizes with downsample, a detection image below 3 x 3, more
 * than PUS_POPUP_LINES_MAX_PIXELS pixels in a frame (pixel indices are 32-bit).  Deterministic (no floating-point
 * atomics): repeated calls and any split of the batch give the same bytes.  No CPU fallback. */
#define PUS_POPUP_LINES_MAX_PIXELS (1LL << 28)
long long pus_popup_lines(int device, int n_frames, const unsigned char* images, int width, int height, int channels,
                          int downsample, int* status, int* counts, float* lines, long long capacity);

/* ---- pop-up session: whole frames, device-resident ------------------------------------------------------------------ */
/* main_3d's per-frame pop-up (main_3d.cpp:417-454 on popup_plane) over a batch of frames in one call, with intermediates kept
 * on the device, scratch reused across runs and no host loop between the stages.  Per frame, in main_3d's order:
 *   1 lines (pus_popup_lines, downsample = fast_edges);  2 edges (pus_popup_edges);  3 the fit, mode 0, on the OPEN segments
 *   (pus_popup_fit_frames);  4 get_plane_equation's actual-index filter on its good flags (popup_plane.cpp:629-635 with
 *   get_ground_edges' actual_plane_indices_inall = {0} u {open_in_connect + 1}, :792-794): open wall s stays good only when
 *   s is one of the frame's open_in_connect values;  5 polygons on the OPEN segments (pus_popup_polygons; the reference's
 *   get_plane_equation calls find_2d_3d_closed_polygon on the list it fits, :551, 607), so their rows are the fit's;
 *   6 clouds of the good rows (pus_popup_clouds) from their cut polygons when walllength_threshold > 0 and their bound ones
 *   otherwise (:821-823), given the images when they are BGR (and with them the 960-wide border rule; a grey session gives
 *   the clouds no images, so colour 0 and no border rule, as the stage call without images);  7 with want_depth the depth map of the good rows'
 *   bound polygons (pus_popup_depth).  Each output equals, bit for bit, what those stage calls give for the same frames
 *   with this glue between them.  A frame without open segments has no good planes and no clouds, not even the ground
 *   (the reference's ground_seg2d_lines.rows() > 0 branch, :553, 645-650).  cloud_projected_plane is not built (it is
 *   always zero on this path, :44, 834).
 * Inputs (each a host or a device pointer, told apart by cudaPointerGetAttributes; host data goes through the session's
 * pinned staging, device data is read in place, ordered on the session's stream): images [n][height][width][channels]
 * (BGR or grey), labels [n][height][width] (ground 255), Ts [n][16] row-major camera-to-world.
 * Per-frame outcomes instead of whole-batch refusals (other frames are unaffected):
 *   status[f]        0 planes popped up (possibly none); 1 the frame's lines are ones pus_popup_edges refuses (more than
 *                    PUS_POPUP_MAX_LINES, or a coordinate not finite): the edge stage is not run for it; 2 more than
 *                    PUS_POPUP_MAX_SEGMENTS open segments.  A frame with a non-zero status has no segments, no good planes
 *                    and no clouds; its fit rows are the one empty ground row of a frame without segments.
 *   line_status[f]   pus_popup_lines' status (0 / 1), line_counts[f] its counts
 *   edge_status[f]   pus_popup_edges' status (0-5), -1 where status is 1
 *   plane_status[p]  per good plane, bit 0: its cloud polygon has more than PUS_POPUP_MAX_VERTICES vertices or a coordinate
 *                    beyond PUS_POPUP_MAX_COORD (checked before the truncation): the plane gets no points and no label
 *                    pixels; bit 1: the same for its bound polygon, which the depth map then does not draw.
 * Outputs, packed in frame order as the stage calls pack them (pus_popup_frames; rows r of frame f run from
 * open_ptr[f] + f to open_ptr[f + 1] + f, row 0 of a frame its ground): the open and connected segments with
 * open_in_connect; per row planes_world, planes_sensor, dist and good after the filter; per row the bound, cut and world
 * polygons (CSR offsets bound_ptr / cut_ptr / world_ptr); good_ptr [n + 1] / good_rows [n_good], the frames'
 * good_plane_indices (row indices within the frame); per good plane its cloud's count and offset into xyz / rgb; labels
 * [n][height][width] and depth [n][height][width] when asked for.
 * Sizing: buffers only grow (by at least half their size), host and device inputs take the same buffers.  A run
 * synchronises with the host four times to read back totals (the line total with the edge scratch, the open / connected
 * segment totals, the good planes with the polygon and box totals, the point total).  The buffers sized by the batch shape
 * never grow again; those sized by these totals grow only when a total exceeds what the buffers hold.  So a run of the
 * same frames as an earlier one performs no cudaMalloc / cudaFree, and neither does one of other frames of the same shape
 * whose totals fit (pus_popup_session_memory counts the allocations).  Deterministic, no floating-point atomics: repeated runs, any split of
 * the batch and reuse across batch sizes give the same bytes.
 * Refused with a message, nothing launched, the session still usable: a NULL session or input, n_frames < 0, and at create
 * a config that the stage calls would refuse (channels, sizes below 4 x 4, odd sizes with fast_edges, or with
 * downsample_poly and labels or depth, kernel sizes below 1, non-finite K / invK) or want_rgb with grey images.
 * A single-threaded object; no CPU fallback. */
typedef void* pus_popup_session;
typedef struct pus_popup_config {
  float K[9], invK[9];                 /* row-major */
  int width, height, channels;         /* fixed for the session; channels 1 (grey) or 3 (BGR) */
  int fast_edges;                      /* popup_plane::use_fast_edges_detection: pus_popup_lines' downsample */
  pus_edge_params edges;               /* as pus_popup_edges */
  float plane_cam_dist_thre;           /* get_plane_equation */
  float ceiling_threshold, walllength_threshold;   /* main_3d: 5.0, 3.0 */
  int downsample_poly;                 /* generate_cloud's and get_depth_map_good's downsample; main_3d: 1 */
  float depth_thre;                    /* generate_cloud's; main_3d: 10.0 */
  int want_rgb, want_labels, want_depth;           /* optional outputs */
} pus_popup_config;
typedef struct pus_popup_frames {
  int n_frames, n_rows, n_good;
  long long n_open, n_connect, n_bound, n_cut, n_world, n_points;
  int *status, *line_status, *line_counts, *edge_status;         /* [n_frames] */
  int *open_ptr, *connect_ptr;                                   /* [n_frames + 1] */
  float *open_segs, *connect_segs;                               /* [n_open][4], [n_connect][4] */
  int* open_in_connect;                                          /* [n_open] */
  float *planes_world, *planes_sensor, *dist;                    /* [n_rows][4], [n_rows][4], [n_rows] */
  int* good;                                                     /* [n_rows] */
  int *bound_ptr, *cut_ptr, *world_ptr;                          /* [n_rows + 1] */
  float *bound2d, *cut2d, *world3d;                              /* [n_bound][2], [n_cut][2], [n_world][3] */
  int *good_ptr, *good_rows, *plane_status, *cloud_counts;       /* [n_frames + 1], [n_good] x 3 */
  long long* cloud_offsets;                                      /* [n_good] */
  float* xyz;                                                    /* [n_points][3] */
  unsigned char *rgb, *labels;                                   /* [n_points][3] (r, g, b); [n_frames][height][width] */
  float* depth;                                                  /* [n_frames][height][width] */
} pus_popup_frames;
int pus_popup_session_create(int device, const pus_popup_config* config, pus_popup_session* out);
int pus_popup_session_destroy(pus_popup_session s);
/* run on this CUDA stream (cudaStream_t as void*); NULL: the session's own stream */
int pus_popup_session_set_stream(pus_popup_session s, void* cuda_stream);
int pus_popup_session_run(pus_popup_session s, int n_frames, const unsigned char* images, const unsigned char* labels,
                          const float* Ts);
/* the last successful run's counts and device pointers (valid until the next run or destroy) */
int pus_popup_session_result(pus_popup_session s, pus_popup_frames* out);
/* copies every output whose pointer in dst is non-NULL (host or device memory, sized from the result's counts) on the
 * session's stream, then synchronises once */
int pus_popup_session_download(pus_popup_session s, pus_popup_frames* dst);
/* device and pinned allocations made so far, and the bytes they hold */
int pus_popup_session_memory(pus_popup_session s, long long* allocations, long long* reserved_bytes);

/* ---- device-resident measurement refresh and polygon re-projection (SURVEY.md 8f.1) -------- */
/* Mapper_mono::update_plane_measurement (pop_planar_slam/src/Mapping.cpp:590-607): after a solve every past
 * frame re-pops its wall planes from its ground segments with the frame's LATEST pose estimate
 * (popup_plane::update_plane_equation_from_seg, popup_plane.cpp:654-705, float32) and stores the sensor-frame
 * plane of every kept observation as the new measurement of its pose-plane factor
 * (Plane3d(Vector4d) normalisation, isam_plane3d.h:59-66; FactorT::set_measurement, Factor.h:203-206).
 * Here the poses are read from the device-resident estimates of the last solve / upload (uploaded first if the
 * graph is not resident), the fit and the factor store run on the device, and only the new measurements come
 * back to refresh the host mirrors (pus_get_measurement):
 *   frame_pose[n_frames]   pose node id of every frame
 *   seg_ptr[n_frames+1], segs, invK   as pus_popup_fit_frames (a malformed seg_ptr is refused before any device work)
 *   map_fid / map_frame / map_row [n_map]   factor id, frame index, plane row inside the frame
 *                                           (0 = ground, 1 + i = segment i: good_plane_indices)
 *   new_meas[n_map*4]      optional copy of the stored measurements */
int pus_refresh_plane_measurements(pus_handle h, int n_frames, const int* frame_pose, const int* seg_ptr,
                                   const float* segs, const float* invK, int n_map, const int* map_fid,
                                   const int* map_frame, const int* map_row, double* new_meas);
/* Resident form of the same sweep (the reference re-pops EVERY past frame after EVERY solve, Mapping.cpp:590-607, while the
 * frames' segment lists never change): pus_refresh_bind uploads the tables once (again whenever frames / factors are added);
 * pus_refresh_run re-pops every bound frame from the device-resident pose estimates and stores the new measurements straight
 * into the device factor store.  new_meas = NULL: nothing returns to the host -- the host mirrors (pus_get_measurement,
 * FactorT::measurement()) are refreshed lazily on their next read or at the next layout rebuild; new_meas != NULL: [n_map][4]
 * out, mirrors refreshed at once.  A structural edit between bind and run is fine as long as the bound frames / factors still
 * exist (the layout-dependent tables are rebuilt by the run).  pus_refresh_bind refuses a malformed seg_ptr as
 * pus_refresh_plane_measurements does. */
int pus_refresh_bind(pus_handle h, int n_frames, const int* frame_pose, const int* seg_ptr, const float* segs, const float* invK,
                     int n_map, const int* map_fid, const int* map_frame, const int* map_row);
int pus_refresh_run(pus_handle h, double* new_meas);
/* Plane3d::project_to_plane (isam_plane3d.h:172-177) over point lists, as Mapper_mono::reproj_to_newplane
 * applies it to every stored polygon vertex (Mapping.cpp:609-632): pts_out[i] = float(project(double(pts_in[i])))
 * onto the current device-resident estimate of plane node plane_of_point[i]. */
int pus_project_to_planes(pus_handle h, int n_points, const int* plane_of_point, const float* pts_in, float* pts_out);

/* ---- plane map: Mapper_mono::processFrame on the device (DESIGN.md section 5.11) ------------------------------------ */
/* A map bound to one solver handle keeps pop_planar_slam's landmark table (Map_plane, PPS/src/Map_plane.h) on the device
 * and maps each frame's good planes into the handle's graph as Mapper_mono::processFrame (PPS/src/Mapping.cpp:401-586) and
 * main_3d's frame loop (PPS/src/main_3d.cpp:366-385, 464-504) do.  Single-threaded, like the handle; it works on the
 * handle's stream.  The caller sets the handle's properties (Mapping.cpp:31-43: LM, mod_batch 1, epsilons x 0.1).
 * There are no defaults: every field of the config is used (capi.PlaneMap has the plane_3d_tum_far.yaml and the
 * Mapping.h:72-94 presets).  Refused at create: a NULL handle or config, a non-finite value, a sigma whose square or
 * inverse square is not a positive finite number, a plane_sigma_dist_mul that makes a pose-plane sigma non-positive. */
typedef void* pus_map;
typedef struct pus_map_config {
  double edge_asso_2ddist, edge_asso_proj, edge_asso_angle, edge_asso_planedist;   /* findClosestPlane's gates */
  int assoc_near_frames;
  double pose_sigmas[6];          /* x y z yaw pitch roll: the prior and odometry noise */
  double plane_sigmas[3];         /* the ground prior's noise */
  double plane_sigma_dist_mul;    /* pose-plane sigma = (clamp(dist, 3, 8) - 1) * mul + 5 */
  double init_wTo[16];            /* the first frame's pose, row-major camera-to-world (main_3d.cpp:368-376) */
  float invK[9];                  /* row-major, for the measurement refresh */
} pus_map_config;
/* one landmark (Map_plane): its plane node, whether that node was removed (pus_remove_node: deteted_by_merge, skipped
 * and never re-projected), the latest observation's descriptor (copy_plane, Map_plane.cpp:11-29) and the first two
 * vertices of its 2-D bound and 3-D world polygons, which are all the association reads (n_* of them stored) */
typedef struct pus_map_landmark {
  int node, deleted, frame_seq_id, frame_plane_indice, good_plane_indice, being_tracked_times;
  double plane_dist_cam;
  int n_bound2d, n_world3d;
  float bound2d[2][2], world3d[2][3];
} pus_map_landmark;
/* One frame's good planes, in one of two forms.  session != NULL: frame `frame` of that pop-up session's last run, read in
 * place on the device (its good rows, planes_sensor, dist, bound2d, world3d and open segments).  Otherwise n_planes planes
 * in arrays, each host or device memory (told apart as the session does): planes_sensor [n][4], dist [n], plane_indice [n]
 * (the plane's row in the frame: 0 ground, 1 + s wall of open segment s), bound_ptr [n + 1] / bound2d [..][2] and
 * world_ptr [n + 1] / world3d [..][3] (CSR), and the frame's n_segs open segments segs [n_segs][4] for the refresh.
 * odom7 (host, x y z qw qx qy qz) is the frame's odometry (temp_pose); NULL takes that of the last pus_map_predict_pose. */
typedef struct pus_map_frame {
  int seq_id;                       /* main_3d's counter */
  const double* odom7;
  pus_popup_session session;
  int frame;
  int n_planes;
  const float *planes_sensor, *dist;
  const int* plane_indice;
  const int* bound_ptr; const float* bound2d;
  const int* world_ptr; const float* world3d;
  int n_segs; const float* segs;
} pus_map_frame;
/* Outputs of one frame; the per-plane arrays (caller-owned host memory, any may be NULL) hold `capacity` entries, in plane
 * order.  landmark: its index; error: the reference's assoc_error (the match error, -1 for a ground match; 0 for a new
 * landmark, and -1 for the plane that loses a dual match to a later one); status: 0 matched, 1 a wall whose bound or world
 * polygon has fewer than two vertices (a new landmark, never matched later: the reference reads past .col(1)), 2 no
 * candidate (new), 3 lost a dual match (new); factor: its pose-plane factor id.  Per frame: pose_node, n_new and the new
 * plane nodes (new_nodes, landmark-index order, room for `capacity`), the solve's LM iteration count (pus_stats). */
typedef struct pus_map_result {
  int capacity;
  int n_planes, pose_node, n_new, lm_iterations;
  int *landmark, *status, *factor, *new_nodes;
  double* error;
} pus_map_result;
int pus_map_create(pus_handle h, const pus_map_config* config, pus_map* out);
/* destroy gives the handle's refresh tables up (unbound): a later map on the same handle starts them afresh */
int pus_map_destroy(pus_map m);
/* main_3d.cpp:366-385 from the handle's device-resident estimates, keyed on the number of MAPPED frames (main_3d keys it on
 * its frame counter, which also counts frames without good planes, and reads all_frames.back() of an empty list there):
 * none -> odometry = prediction = the config's initial pose; one -> zero odometry; more -> last.ominus(previous).  The
 * prediction is last.oplus(odometry); T16 (host or device memory) receives its wTo() as row-major float, ready for
 * pus_popup_session_run's Ts; odom7 (host, may be NULL) the odometry, which the next pus_map_process_frame takes when its
 * odom7 is NULL. */
int pus_map_predict_pose(pus_map m, float* T16, double* odom7);
/* One frame, in main_3d's order: 1 association (findClosestPlane and the one-to-one rule, against the estimate
 * last.oplus(odom), the identity on the first frame); 2 graph edits, ids in insertion order: the pose node, the prior at
 * odom (first frame) or the odometry factor, the new plane nodes in landmark order (initialised at their measurement
 * through the estimate's oTw), then per plane the ground prior (0,0,-1,0) for a new ground landmark and the pose-plane
 * factor, noise as isam::Covariance forms it (include/popup_noise.hpp);  3 copy_plane;  4 pus_batch_optimize when
 * seq_id % 5 == 0, else pus_update;  5 the landmarks' stored 3-D vertices projected onto their planes' new estimates
 * (as pus_project_to_planes);  6 the measurement refresh (pus_refresh_run) over every mapped frame, whose tables the map
 * appends to (the frame's open segments, its pose, its planes' factor and row) -- a pus_refresh_bind on the handle
 * afterwards takes the tables away, and the map then refuses further frames.  A frame without planes changes nothing.
 * Refused with a message before any edit, map and handle unchanged: NULL arguments, too small a capacity, a session frame
 * out of range, a non-finite value among those read (planes, dist, the first two vertices, the segments), a
 * plane_indice outside 0..n_segs, more than one ground plane, a frame with planes but no open segments (as
 * pus_refresh_bind), malformed CSR offsets, no odometry, a removed last pose.  An edit that fails removes the nodes the
 * frame added (with their factors) and leaves the map as it was; a failing solve leaves the edits in place.  Deterministic: repeated runs, the session and array forms, host and device
 * inputs give the same bytes. */
int pus_map_process_frame(pus_map m, const pus_map_frame* in, pus_map_result* out);
/* the landmark table (capacity records; out = NULL is a size query); returns the number of landmarks */
int pus_map_landmarks(pus_map m, int capacity, pus_map_landmark* out);

/* ---- weighted errors and the stacked Jacobian at the current estimate ---------------------------- */
/* Evaluated on the device, one thread per live factor, with the residual and Jacobian code the solver linearises with.
 * Rows follow the factor order and columns the node order of pus_factor_row / pus_node_start (Slam::update_starts
 * Slam.cpp:59-67, jacobian_partial :395-432).  Each call first re-uploads the graph if its topology, host values or
 * measurements changed since the last upload, as pus_project_to_planes does; otherwise it reads the device-resident
 * estimate of the last solve.  The outputs do not depend on the linear solver (PCG and direct handles agree bit for bit)
 * and repeated calls are bit-identical (no floating-point atomics; the sums below reduce in a fixed order).
 * A graph without live factors, a bad factor id or too small a capacity fails with a message. */
/* VectorXd Slam::weighted_errors(ESTIMATE)  Slam.cpp:254-264: Factor::error of every live factor, stacked.  Returns the
 * number of rows (the sum of the live factors' dims); out = NULL is a size query. */
long long pus_weighted_errors(pus_handle h, double* out, long long capacity);
/* VectorXd Factor::error(ESTIMATE)  Factor.h:67-77 of n factors: their rows packed in the order of fids.  Returns the
 * total number of rows. */
int pus_factor_errors(pus_handle h, int n, const int* fids, double* out);
/* SparseSystem::num_rows() / num_cols() of Slam::jacobian(): the sum of the live factors' dims and of the live nodes' dims
 * (host only). */
int pus_jacobian_dims(pus_handle h, long long* rows, long long* cols);
/* SparseSystem Slam::jacobian()  Slam.cpp:379-432 at the current estimate, as CSR: row_ptr [rows + 1], col_idx / values
 * [nnz], rhs [rows] = Jacobian::rhs() = minus the residual rows (Jacobian.h:97-98).  Within a row the columns ascend and
 * zeros stay stored ("0-entries not omitted", Slam.cpp:425).  Any output may be NULL; cap_nnz = 0 is a size query.
 * Returns nnz.  The blocks follow pus_set_jacobian_mode, as the solve does:
 *   mode 0 (default)  closed forms; they agree with the reference's central differences to its O(eps^2) truncation error
 *                     (about 1e-8 relative);
 *   mode 1            the reference's central differences (numericalDiff, eps = 1e-4) through the Euler round trip of the
 *                     linearisation point, as Factor::jacobian forms them.  rhs is then the residual at the round-tripped
 *                     point, as upstream (it differs from -pus_weighted_errors in the last bits).
 *                     This is Slam::jacobian()'s default branch, jacobian_partial.  With force_numerical_jacobian the
 *                     reference runs jacobian_numerical_columnwise instead, which has the same values but omits exact zeros
 *                     and returns +residual as its rhs (Slam.cpp:365, 375); the export does not follow that branch.
 * row_ptr / col_idx depend only on the graph's structure and are built once per layout, on the device. */
long long pus_jacobian(pus_handle h, int* row_ptr, int* col_idx, double* values, double* rhs, long long cap_nnz);
/* double Slam::normalized_chi2()  Slam.cpp:287-289: chi2 / (rows - columns) */
int pus_normalized_chi2(pus_handle h, double* out);
/* double Slam::local_chi2(int last_n)  Slam.cpp:270-285: the sum of squares of the weighted errors of the last_n most recent
 * live factors (all of them when last_n exceeds their number; 0 when last_n <= 0) */
int pus_local_chi2(pus_handle h, int last_n, double* out);

/* ---- marginal covariances (isam::Covariances, Covariances.h:58-110; DESIGN.md section 5.4) ---------------------------- */
/* Sigma = (J^T J)^-1 at the current estimate, undamped (lambda = 0), where J is the stacked whitened, robustified Jacobian
 * that pus_jacobian exports: the same column order and tangent parameterisation as pus_node_start, and it follows
 * pus_set_jacobian_mode.  This is what iSAM returns right after Slam::update() with mod_batch = 1 (Optimizer::relinearize
 * factors undamped at the pre-step point, and Covariances reads that R).  After batch_optimization() iSAM's R is its last
 * damped trial factor, so its covariances differ from these by O(lambda); that is not reproduced.
 * Only a handle with pus_set_linear_solver(h, 2) and pus_set_direct_ordering(h, 1) recovers covariances; every other handle
 * (PCG, dense kind 1, band in insertion order, and hence a pus_span_* handle) is refused with a message naming those calls.
 * The first call at an estimate linearises, factors the reduced system undamped and inverts it on L's tile pattern by
 * selected inversion (about the cost of one factorization); the Sigma tiles stay on the device, and later calls read them
 * until a solve, pus_init_*, a measurement change, a structural edit, pus_set_robust or pus_set_jacobian_mode.  The calls
 * never change the estimate, the trace or the solver's statistics other than kernel_ms.  A non-positive pivot (J^T J not
 * positive definite, e.g. no pose prior: the gauge is free) fails the call with a message and stores nothing.  The Sigma tiles
 * and the selected-inversion lists count against the band budget of 8 GiB together with the factorization; an over-budget
 * graph is refused at the first call with the need stated, and nothing is launched.  Results are bit-identical across team
 * sizes, barrier kinds and repeated calls (no floating-point atomics, fixed summation orders).
 * Cost: the blocks of kept unknowns (poses, bordered planes) whose tile is stored, and every plane's own block, are read
 * from Sigma (an eliminated plane's block sums over its observer pairs).  Any other block (two distant poses, a pose and a
 * plane it does not co-observe, two eliminated planes) costs one pair of triangular solves with the factor per column of
 * its right-hand node (6 for a pose, 3 for a plane), shared by every block of the call with that right-hand node. */
/* Each node's own block (6 x 6 for a pose, 3 x 3 for a plane), full, row-major, packed in ids order; n may be every live
 * node.  Returns the number of doubles written, or < 0. */
int pus_marginal_covariances(pus_handle h, int n, const int* ids, double* out);
/* The cross blocks Sigma_ab, dim(a) x dim(b) row-major, of the pairs (id_pairs[2 k], id_pairs[2 k + 1]), packed in pair
 * order (Covariances::access).  Returns the number of doubles written, or < 0. */
long long pus_covariance_blocks(pus_handle h, int n_pairs, const int* id_pairs, double* out);

/* ---- one graph spanning several ranks (SURVEY.md 8e, second bullet) --------------------------- */
/* Every rank holds the whole graph (build it identically on each) and runs its own persistent kernel; the PCG
 * phases -- the two Schur sweeps, the pose phase, the preconditioner, the dot products -- are split over the CTAs of
 * ALL ranks.  The vectors they exchange (plane partial sums, p, q, r, x, z, the coarse residuals, the reduction
 * partials) sit in one "mirror arena" per rank; owners store their entries into every peer's arena through
 * NVLink peer memory and the ranks meet at a cross-rank barrier (system-scope atomics) where the single-GPU path
 * has its team barrier -- no host round trip and no NCCL call inside the solve.  Linearisation, the Schur
 * set-up and the LM update are replicated, so all ranks take identical decisions and end with identical estimates.
 *   pus_span_export   uploads the graph if needed and writes the 64-byte CUDA IPC handle of this rank's arena
 *   pus_span_connect  opens the peers' handles (handles = world x 64 bytes, in rank order; own entry ignored)
 *   pus_span_optimize batch_optimization() of the spanning graph; call on every rank
 *   pus_span_disconnect closes the peer mappings (also done by pus_destroy)
 * pus_span_emulate_optimize runs the same protocol with `world` handles on ONE device (one CTA team per handle inside
 * a single launch) -- the test vehicle for the protocol on a single GPU. */
int pus_span_export(pus_handle h, void* ipc_handle_64);
int pus_span_connect(pus_handle h, int rank, int world, const void* handles);
int pus_span_optimize(pus_handle h, int* iterations);
int pus_span_disconnect(pus_handle h);
int pus_span_emulate_optimize(pus_handle* handles, int world, int* iterations);

/* ---- graph text I/O (SURVEY.md 8f.4; host only) ---------------------------------------------- */
/* Slam::save (ISAM/isamlib/Slam.cpp:84-89 -> Graph::write, Graph.h:120-131): every factor, then every node, one per
 * line: "<Factor name> <node ids> <measure> {sqrtinf upper triangle, row-wise, comma separated}" (Factor.h:148-155,
 * 169-190, 208-211) and "<Type>_Node <id> <value>" (Node.h:148-153); Pose3d prints "(x, y, z; yaw, pitch, roll)"
 * (Pose3d.h:169-172), Plane3d "(a, b, c; d)" (isam_plane3d.h:190-192).  The plane prior keeps the reference's
 * name "Pose3d_Factor" (isam_plane3d.h:438).  precision <= 0 = the stream default of the reference (6 digits). */
int pus_save_graph(pus_handle h, const char* path, int precision);
/* The 3-D part of the iSAM dataset grammar (ISAM/isam/Loader.cpp:316-392): EDGE3 i j x y z roll pitch yaw [21
 * sqrt-information entries, rotational block re-ordered] with the reversal of edges that point backwards and the
 * 100*I prior on the first pose (Loader.cpp:48-64), POSE3D_INIT; EDGE3_INIT / POSE3D_TRUE / EDGE3_TRUE / SOLVE are
 * skipped as upstream; the 2-D and stereo keywords are rejected.  Nodes are left to the factors' initialize().
 * n_poses / n_factors (optional) receive what was added. */
int pus_load_isam_dataset(pus_handle h, const char* path, int* n_poses, int* n_factors);

/* ---- debug / test hooks ----------------------------------------------------------------- */
/* copy a named device buffer of the last upload/solve to the host as doubles
 * ("Hpp","gp","Hll","gl","W","Wt","Hoff","Minv","delta", ...). Returns element count, <0 if unknown. */
long long pus_debug_fetch(pus_handle h, const char* name, double* out, long long capacity);
/* run single stages on the uploaded graph: 0 linearise at the current linpoint (fills Hpp..W),
 * 1 build Schur preconditioner for `lambda`, 2 one solve for `lambda` (fills "delta"),
 * 3 y = S*x for the vector previously stored with pus_debug_store("x").
 * Direct linear-solver mode only: 4 stop after the assembly of S ("Sdir"), 1 also factors it ("Ldir");
 * 5 factors the S stored with pus_debug_store("Sdir") (no linearisation, `lambda` unused) and, unless a pivot is not
 * positive, solves S x = b for the vector stored with pus_debug_store("b"), leaving x in "x".  pus_debug_fetch("dflag")
 * returns one value: 1 when the last factorization met a non-positive pivot, else 0.  Stage 5 is refused for a PCG handle. */
int pus_debug_run_stage(pus_handle h, int stage, double lambda);
/* copy host doubles into a named device buffer; "Sdir" (direct mode, after pus_upload) takes a dense row-major (6 N)^2
 * matrix, of which the lower triangle is laid out as the assembly lays out S (padding rows are identity); it refuses
 * any other element count */
long long pus_debug_store(pus_handle h, const char* name, const double* in, long long count);

#ifdef __cplusplus
}
#endif
#endif /* POPUP_GPU_H */
