/* immesh_b200 -- C ABI of the H100-native (sm_90a) ImMesh localization + meshing hot path.
 *
 * The reference (hku-mars/ImMesh) has no plugin / FFI layer; this header cuts the drop-in
 * boundary at the C++ seams its ROS node calls.  Every entry point names the reference
 * function it replaces (paths relative to the reference repository).  All buffers are plain
 * caller-owned host arrays (row-major); handles own all device memory; no exceptions cross the
 * boundary; every function returns 0 on success or a negative IMMESH_E_* code.  Calls on one
 * handle must be serialised by the caller (exactly as the reference serialises its LIO thread
 * and its mesh frames); different handles may be used concurrently.
 */
#ifndef IMMESH_B200_H_
#define IMMESH_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define IMMESH_OK 0
#define IMMESH_E_INVALID (-1)  /* bad argument */
#define IMMESH_E_CUDA (-2)     /* CUDA runtime failure (see immesh_last_error) */
#define IMMESH_E_CAPACITY (-3) /* a device pool / hash table overflowed */
#define IMMESH_E_NO_DEVICE (-4)
#define IMMESH_E_RANGE (-5)    /* coordinate outside the representable key range */

#define IMMESH_STATE_DOUBLES 348 /* rot_end[9] pos_end[3] vel_end[3] bias_g[3] bias_a[3] gravity[3] cov[18*18]
                                    = StatesGroup, include/common_lib.h:199-288 */
#define IMMESH_ITER_STATS_DOUBLES 63 /* HTH[36] HTz[6] n_match total_residual solution[18] converged */
#define IMMESH_MAP_DUMP_COLS 45
#define IMMESH_PTPL_DOUBLES 31 /* point[3] normal[3] center[3] d plane_var_upper[21]  (struct ptpl, src/voxel_loc.hpp:63-73) */

typedef struct immesh_lio immesh_lio_t;
typedef struct immesh_mesh immesh_mesh_t;
typedef struct immesh_voxelgrid immesh_voxelgrid_t;
typedef struct immesh_imu immesh_imu_t;

/* Parameters of Voxel_mapping that the path reads (src/voxel_mapping.hpp:149-191,
 * read_ros_parameters src/voxel_mapping_common.cpp:625-707). */
typedef struct immesh_lio_config {
    double voxel_size;         /* voxel/voxel_size -> m_max_voxel_size */
    int max_layer;             /* voxel/max_layer */
    int layer_init_size[5];    /* voxel/layer_init_size */
    int max_points_size;       /* voxel/max_points_size */
    double min_eigen_value;    /* voxel/min_eigen_value */
    double dept_err, beam_err; /* voxel/dept_err, voxel/beam_err */
    double ext_R[9], ext_T[3]; /* mapping/extrinsic_R, extrinsic_T (LiDAR -> IMU) */
    int max_iteration;         /* max_iteration (NUM_MAX_ITERATIONS), <= 8 */
    int calib_laser;           /* preprocess/calib_laser */
    /* capacities of the device-resident map (0 = defaults) */
    int hash_capacity_log2;    /* root-voxel hash slots = 2^this          (default 22) */
    int max_nodes;             /* octree node / plane records              (default 4 Mi) */
    int max_chunks;            /* 8-point storage chunks (512 B each)      (default 4 Mi) */
    int max_scan_points;       /* largest scan handed to any call          (default 2 Mi) */
} immesh_lio_config;

/* ---- localization handle: owns the VoxelMap (m_feat_map) and the filter state ------------------------ */
int immesh_lio_create(const immesh_lio_config* cfg, immesh_lio_t** out);
int immesh_lio_destroy(immesh_lio_t* h);
int immesh_lio_set_state(immesh_lio_t* h, const double* state /*[348]*/);
int immesh_lio_get_state(immesh_lio_t* h, double* state /*[348]*/);

/* ImuProcess::Forward_without_imu (src/IMU_Processing.cpp:486-553): constant-velocity prediction of the
 * state and its covariance, used when imu_en is false. */
int immesh_lio_predict(immesh_lio_t* h, double dt, double cov_gyr, double cov_acc);

/* Voxel_mapping::voxel_map_init + buildVoxelMap (src/voxel_mapping.cpp:1243-1281, :110-151):
 * first-scan map construction from the full-resolution body-frame scan, at the current state. */
int immesh_voxelmap_build(immesh_lio_t* h, const float* body_xyz /*[n][3]*/, int n);

/* Voxel_mapping::lio_state_estimation (src/voxel_mapping.cpp:1284-1652): all IESKF iterations on the
 * down-sampled body-frame scan; the propagated state is the handle's state on entry.  The whole loop
 * (BuildResidualListOMP + Jacobian + H^T R^-1 H reduction + 18x18 solve + convergence logic) runs on the
 * device without host round trips.  IMMESH_E_RANGE: a coordinate outside the key range, or normal-equation sums beyond the 2^-20 fixed
 * point (a term of 1e10 or more, or a thread's sum of 2^36 or more -- which threads sum which points depends on the GPU's SM count);
 * the state is then undefined and should be restored by the caller. */
int immesh_lio_estimate(immesh_lio_t* h, const float* body_xyz /*[n][3]*/, int n, int* iters_run);

/* Voxel_mapping::map_incremental_grow, VoxelMap part (src/ImMesh_mesh_reconstruction.cpp:387-408 ->
 * updateVoxelMap src/voxel_mapping.cpp:320-354) on the scan last given to immesh_lio_estimate. */
int immesh_voxelmap_update(immesh_lio_t* h);

/* predict + estimate + update for one scan in one call (one H2D copy, one stream, no intermediate sync).
 * dt <= 0 skips the prediction.  state_out may be NULL. */
int immesh_lio_step(immesh_lio_t* h, const float* body_xyz, int n, double dt, double cov_gyr, double cov_acc,
                    double* state_out /*[348] or NULL*/, int* iters_run /*or NULL*/);

/* same, with the scan already resident in device memory (d_body_xyz must stay valid until the next call on h) */
int immesh_lio_step_dev(immesh_lio_t* h, const float* d_body_xyz, int n, double dt, double cov_gyr, double cov_acc,
                        double* state_out, int* iters_run);

/* Pipelined form (the reference runs LIO and meshing concurrently: LIO thread || mesh thread pool, SURVEY 2.2):
 * immesh_lio_step_async queues a scan on the localization stream and returns; immesh_lio_wait blocks until everything
 * queued has finished and returns the latest state.  on_device != 0: body_xyz is a device pointer. */
/* Host buffers: page-locked memory (cudaMallocHost / cudaHostRegister) is read by the copy engine directly and must stay
 * unchanged until the matching wait; pageable memory is staged through the handle's pinned slots at once. */
int immesh_lio_step_async(immesh_lio_t* h, const float* body_xyz, int n, int on_device, double dt, double cov_gyr, double cov_acc);
/* same with the point COUNT device resident too (d_n: device pointer to an int <= n_max, read when the step executes): the scan
 * produced by a device front-end is localised without a host round trip of its size */
int immesh_lio_step_async_dev_n(immesh_lio_t* h, const float* d_body_xyz, int n_max, const int* d_n, double dt, double cov_gyr, double cov_acc);
int immesh_lio_wait(immesh_lio_t* h, double* state_out /*[348] or NULL*/, int* iters_run /*or NULL*/);
int immesh_lio_enqueue_memset(immesh_lio_t* h, void* d_buf, size_t bytes); /* benchmark helper: in-stream L2 flush */

/* Multi-GPU (one process per GPU): shard this handle's VoxelMap by root-voxel key over `nranks` ranks.  Every rank is
 * given the same scans; a rank matches / updates only the root voxels it owns, and the IESKF iterations exchange two
 * integer all-reduces over NCCL (per-point "own-voxel matched" bits, then the 58 fixed-point normal-equation sums), so
 * every rank ends each scan with the bit-identical state of the single-GPU run.  unique_id128: bytes produced by
 * immesh_comm_unique_id on rank 0 and distributed by the caller (e.g. torch.distributed broadcast). */
int immesh_comm_unique_id(char* out128);
int immesh_lio_shard(immesh_lio_t* h, int rank, int nranks, const char* unique_id128);
/* Transport of a sharded handle's exchanges: 0 = handle not sharded, 1 = NCCL collectives, 2 = peer windows.  With peer
 * windows (the default when the ranks' GPUs can map each other's memory through CUDA IPC / NVLink; IMMESH_SHARD_NCCL=1 in
 * the environment forces NCCL) there is no collective call: the kernel that produces the data stores it directly into
 * the consumer ranks' windows and raises an epoch flag, the consuming kernel waits on the flags -- the NCCL communicator
 * is then only used once, to exchange the IPC handles. */
int immesh_lio_shard_transport(immesh_lio_t* h);
int immesh_mesh_shard_transport(immesh_mesh_t* h);
/* Same for the mesher (its own communicator: use a second unique id).  Every rank is given the same frames and runs the
 * vertex append itself (replicated: identical vertex ids everywhere); the per-voxel stage -- dilation, triangulation
 * (mesh_rec_geometry.cpp:174-295), pull, commit -- runs only for the mesh voxels the rank owns.  Two all-gathers per frame
 * exchange (i) the smoothed vertex positions written by the dilations and (ii) the new facets with their flip-priority
 * words plus the removals, which every rank then applies to its replica of the triangle store, so that all replicas hold
 * the single-GPU facet set after every frame. */
int immesh_mesh_shard(immesh_mesh_t* h, int rank, int nranks, const char* unique_id128);

/* BuildResidualListOMP (src/voxel_mapping.hpp:103-105, src/voxel_mapping.cpp:153-245) as a stand-alone call at
 * the current state: fills, for every accepted match in scan order, its scan index, octree layer and the ptpl
 * payload.  Returns the number of matches in *n_out (written entries are capped by cap). */
int immesh_residual_build(immesh_lio_t* h, const float* body_xyz, int n, int* index_layer /*[cap][2]*/,
                          double* ptpl /*[cap][31]*/, int cap, int* n_out);

/* The three free functions of src/voxel_mapping.hpp:80-105 on caller-built Point_with_var lists (what the shim in
 * immesh_b200/csrc/immesh_shim.hpp forwards to).  pts_world: m_point (insert path) / m_point_world (lookup path),
 * var9: m_var row-major, pts_body: m_point of the lookup path.  The caller's order is kept (updateVoxelMap expects
 * its input already sorted by var_contrast).
 * The insert calls (_build_pv, _update_pv) store every world point as float, as the reference's Point_with_var lists are filled
 * from pcl::PointXYZI clouds at every call site: pts_world is rounded to float on entry, so a map built from doubles equals the map
 * built from their float roundings.  The lookup call (_residual_build_pv) uses pts_world as given, in double. */
int immesh_voxelmap_build_pv(immesh_lio_t* h, const double* pts_world /*[n][3]*/, const double* var9 /*[n][9]*/, int n);
int immesh_voxelmap_update_pv(immesh_lio_t* h, const double* pts_world /*[n][3]*/, const double* var9 /*[n][9]*/, int n);
int immesh_residual_build_pv(immesh_lio_t* h, const double* pts_body, const double* pts_world, const double* var9, int n,
                             int* index_layer /*[cap][2]*/, double* ptpl /*[cap][31]*/, int cap, int* n_out);

/* diagnostics used by the parity tests */
int immesh_lio_iter_stats(immesh_lio_t* h, int iter, double* out /*[63]*/);
int immesh_lio_matches(immesh_lio_t* h, int* plane_layer /*[n] layer or -1*/, int n);
int immesh_lio_match_nodes(immesh_lio_t* h, int* plane_node /*[n] plane record index or -1*/, int n);
/* canonical dump of the VoxelMap (roots by ascending key, nodes in pre-order), 45 doubles per node */
int64_t immesh_voxelmap_dump(immesh_lio_t* h, double* rows, int64_t cap_rows);
int immesh_voxelmap_counts(immesh_lio_t* h, int64_t* out /*[4]: roots, nodes, chunks_in_use, error_flags*/);

/* Long runs: the VoxelMap's pools (root hash, node / plane records, 8-point chunks) are sized at create time by
 * immesh_lio_config; these calls enlarge them on a live handle.  A grown handle computes exactly what a handle created at the
 * larger capacities computes.  The per-scan buffers (max_scan_points) do not grow.
 * capacity: out = [root slots, roots, node records, nodes used, chunks, chunks in use, device bytes of the handle, growths so far].
 *   Blocking: waits for the work queued on h.
 * reserve: grow to at least these capacities (<= 0 or below the current one: keep; root slots are rounded up to a power of two).
 *   Never shrinks.  Blocking: drains the steps queued on h first.  Fails with IMMESH_E_CAPACITY (beyond 2^30 records of a pool --
 *   the ids are 32-bit --, above the set_growth ceiling, or out of device memory) or IMMESH_E_CUDA, immesh_last_error() naming the
 *   pool; the handle is then exactly as before.  A sharded handle: IMMESH_E_INVALID.
 * set_growth: max_bytes > 0 turns on automatic growth -- before every step (immesh_voxelmap_build / _update, the *_pv inserts,
 *   immesh_lio_step*, immesh_lio_step_async*) the pools are checked against the use of the last finished step and doubled while
 *   their headroom is short (INTEGRATION.md, "Long runs"); max_bytes is a ceiling on the handle's device bytes.  0: off (the
 *   default); a step then does nothing it did not do before.  A step that overflows anyway returns IMMESH_E_CAPACITY as without
 *   growth. */
int immesh_lio_capacity(immesh_lio_t* h, int64_t* out /*[8]*/);
int immesh_lio_reserve(immesh_lio_t* h, int64_t root_slots, int64_t nodes, int64_t chunks);
int immesh_lio_set_growth(immesh_lio_t* h, int64_t max_bytes);

/* Local map: a cube that follows the sensor, and the eviction of the root voxels it leaves behind, so that the VoxelMap of a drive
 * that keeps reaching new ground stays bounded.  Opt-in and off by default; while it is off (and nothing was evicted) no output,
 * launch sequence or captured graph changes.
 * Box rule: Voxel_mapping::laser_map_fov_segment (src/voxel_mapping_common.cpp:214-288) in the reference's own types -- pos_end
 *   double, the box vertex_min / vertex_max float, dist_to_map_edge float, thresholds mov_threshold * det_range in float, and
 *   mov_dist = max((cube_len - 2 mov det) * 0.5 * 0.9, det (mov - 1)) (:256).  The first evaluation places the box around the pose
 *   (:227-239); each later evaluation that moves it removes, for each axis that moved, the old box with that axis narrowed to the
 *   slab it gave up (:257-278).
 * When: once per scan at the state the scan's IESKF starts from -- after the prediction (for the IMU chain: after UndistortPcl),
 *   before the first match -- by immesh_lio_estimate and the immesh_lio_step* entry points; immesh_voxelmap_build and the IMU chain's
 *   first scan evaluate it at the building scan's pose, which places the box.  The *_pv calls never evaluate it.
 * What is evicted: a root voxel whose centre (the root node's voxel centre, double) lies in a removed box, the float edges widened
 *   to double, half-open min <= c < max as ikd-Tree's Delete_Point_Boxes (include/ikd-Tree/ikd_Tree.cpp:826-827).  Its whole octree
 *   goes: the chunks back to the chunk pool, the node records onto a free stack that new nodes are taken from first, its hash slot
 *   becomes a tombstone.  A root created there later is a fresh root, exactly as on a first visit.  A run with the local map equals
 *   the oracle run with the same eviction (state, match sets, canonical dump); node ids may differ, as between any two runs.
 * Tombstones: when those left by the last finished step exceed 1/8 of the root slots, the next step first drains the handle and
 *   rebuilds the root hash at its size (whatever immesh_lio_set_growth says).  Growth counts tombstones as occupied slots and the
 *   free node records as unused.
 * local_map: cube_len > 0 turns the automatic rule on (the reference's values: cube_side_length, det_range 300, mov_threshold 1.5);
 *   cube_len = 0 turns it off.  Drains the handle; the box is placed at the next evaluation.  A non-finite or non-positive value, or
 *   a sharded handle: IMMESH_E_INVALID; immesh_lio_shard refuses a handle that ever used the local map or evict_boxes.  cube_len <= 2 mov det is allowed
 *   (the reference only warns): the box then moves on every scan.
 * evict_boxes: evicts the root voxels whose centre lies in one of n boxes [n][6] (min xyz, max xyz), by the same rule; queued in
 *   stream order behind the steps already queued (the Delete_Point_Boxes analogue); `boxes` is copied before the call returns.  A NaN edge or a sharded handle: IMMESH_E_INVALID.
 * local_map_state: blocking.  box = the current box (min xyz, max xyz); stats = [box placed, moves, roots evicted, node records
 *   freed, chunks freed, live tombstones, hash rebuilds that dropped tombstones, free node records]. */
int immesh_lio_local_map(immesh_lio_t* h, double cube_len, float det_range, float mov_threshold);
int immesh_voxelmap_evict_boxes(immesh_lio_t* h, const float* boxes /*[n][6]*/, int n);
int immesh_lio_local_map_state(immesh_lio_t* h, float* box /*[6]*/, int64_t* stats /*[8]*/);

/* pubPlaneMap(m_feat_map, voxel_pub, state.pos_end) (src/voxel_mapping.cpp:947-1159), called after voxel_map_init and after every
 * map_incremental_grow (:1899-1900, :1975-1976): the markers of the planes refitted since the last call, one row per pubPlane call
 * (:919-945), with the reference's walk -- a root whose m_is_update flag is set is published and its children wait for a later
 * call; else each child with the flag; else each grandchild with octo_state 0 and the flag, published only when planar (radius
 * not scaled by 1.25), a non-planar one keeping its flag; deeper layers never.  Every flag published is cleared.
 * Row = IMMESH_PLANE_MARKER_COLS doubles:
 *   kx ky kz path layer id | px py pz nx ny nz | radius min_eig trace alpha
 *   key and path as in immesh_voxelmap_dump; id: the node's record index (stable while the node lives, unique per handle; the
 *   reference's g_plane_id counter is not reproduced); p / n: Plane::m_p_center, the float centre and normal of the node's last
 *   PLANAR fit (zeros if it never was one); radius: the float pubPlane receives (1.25 m_radius at layers 0 and 1, m_radius at
 *   layer 2); min_eig: m_min_eigen_value; trace: (pv00 + pv11) + pv22 of m_plane_var (0 for a non-planar fit); alpha: 1 if planar.
 *   The node colours with mapJet(pow(min(trace, 0.25) / 0.25, 0.2), 0, 1) and builds the marker with its own pubPlane (:978-990).
 * Rows are in ascending root key (the dump's order), then in the reference's child order.  Only roots under which a plane was
 * fitted since the last call, or whose markers were held back by it, are visited.  Blocking: waits for the work queued on h.
 * counts (or NULL) = [plane, sub-plane, sub-sub-plane, update counts as printed by the reference (:1154-1158), roots walked];
 * they cover the roots walked, so a non-planar layer-2 flag, which the reference counts as a sub-sub plane again on every call,
 * is counted only while its root is visited.
 * *n_out > cap: returns IMMESH_E_CAPACITY with *n_out = rows needed and nothing consumed (cap = 0: a pure count query).
 * A sharded handle publishes the roots it owns. */
#define IMMESH_PLANE_MARKER_COLS 16
int immesh_voxelmap_plane_markers(immesh_lio_t* h, double* rows /*[cap][16] or NULL*/, int cap, int* n_out, int64_t* counts /*[5] or NULL*/);

/* The two point-cloud publishers that follow map_incremental_grow (src/voxel_mapping.cpp:1983-1995).  Rows are float x y z
 * intensity (PointXYZI as the reference publishes it), world frame = RGBpointBodyToWorld (src/voxel_mapping_common.cpp:168-189):
 * (float) of R (R_ext p + t_ext) + t in double with the handle's CURRENT state (what the reference's publishers read); the
 * reference's extra multiply by _gravity_correct_rotM is the identity and is skipped, which can change at most the sign of a zero.
 * Both calls block: they wait for the work queued on h, the pipelined steps included.  *n_out > cap returns IMMESH_E_CAPACITY with
 * *n_out = rows needed (cap = 0: a pure count query; rows may then be NULL).
 * Validity: the rows of immesh_lio_effect_cloud, and those of immesh_lio_registered_cloud with pts == NULL, belong to the last
 * IESKF run (immesh_lio_estimate or any immesh_lio_step* entry point).  Before any run, and after immesh_voxelmap_build, the effect
 * cloud has 0 rows (the reference's m_effct_feat_num is 0) and pts == NULL returns IMMESH_E_INVALID.  immesh_residual_build and the
 * three *_pv calls overwrite the per-scan buffers: the effect cloud and pts == NULL then return IMMESH_E_INVALID, naming the call,
 * until the next run.  immesh_voxelmap_update changes neither.
 * A sharded handle returns the effect rows of the matches it contributed (their union over the ranks, ordered by scan index, is the
 * single-GPU cloud); its registered cloud is the same on every rank. */
#define IMMESH_SCAN_PUB_COLS 4
/* publish_effect_world (src/voxel_mapping_common.cpp:535-547, /cloud_effected): the scan points matched in the LAST IESKF iteration
 * (m_laserCloudOri, ptpl order = ascending scan index, src/voxel_mapping.cpp:1372-1392), intensity = (float)sqrt(R_inv), the
 * point's IESKF weight (:1527, :1558), as stored when the residual was formed.  scan_index (or NULL): each row's index in the scan. */
int immesh_lio_effect_cloud(immesh_lio_t* h, float* rows /*[cap][4]*/, int32_t* scan_index /*[cap] or NULL*/, int cap, int* n_out);
/* publish_frame_world (src/voxel_mapping_common.cpp:595-614, /cloud_registered, publish/pub_point_skip): points 0, point_skip,
 * 2 point_skip, ... of pts ([n][stride] floats, x y z in the first three columns; on_device != 0: a device pointer) in the world
 * frame; intensity = pts[i * stride + intensity_col], or 0 when intensity_col < 0.  A host buffer is copied to a staging buffer of
 * its own; the scan the handle localised is left as it is.
 * pts == NULL (dense_map_en = 0): the down-sampled scan the handle last localised, read where the run read it (a caller-owned
 * device scan must still hold it), intensity 0 -- the plain front-end chains do not carry intensity (PCL's VoxelGrid averages it;
 * immesh_lio_frontend_cloud publishes it after the _i chains); n, stride, intensity_col and on_device are then ignored.
 * point_skip <= 0 (the reference would loop forever), stride < 3 or intensity_col >= stride: IMMESH_E_INVALID. */
int immesh_lio_registered_cloud(immesh_lio_t* h, const float* pts, int n, int stride, int intensity_col, int on_device,
                                int point_skip, float* rows /*[cap][4]*/, int cap, int* n_out);

/* Scan feed: what the reference publishes after every scan (publish_odometry, kitti_log, dump_lio_state_to_log, publish_path,
 * publish_mavros, /cloud_registered, /cloud_effected; src/voxel_mapping.cpp:1963-2002), recorded on the device in stream order as
 * part of each scan's launch sequence, so that a node on the queued chain can publish scan k after scan k + 1 is queued, without
 * draining.
 * immesh_lio_feed_enable(h, cfg) drains h, drops its captured launch sequence and allocates the rings once; numbering restarts at
 *   scan 1.  cfg == NULL turns the feed off and frees the rings; while it is off, nothing is launched or recorded for it.
 *   max_scans >= 1: header and state ring; max_rows: row ring (>= 1 when effect or registered is set); effect 0/1; registered 0 (none),
 *   1 (the down-sampled scan, dense_map_en 0) or 2 (the full scan, dense_map_en 1); point_skip >= 1 (publish/pub_point_skip).
 *   Other values, or a sharded handle: IMMESH_E_INVALID.  immesh_lio_shard refuses a handle with the feed on.
 * Every call of immesh_lio_step, _step_dev, _step_async, _step_async_dev_n, _step_async_raw, _raw_i, _imu, _imu_i, _depth and _depth_imu records
 * one scan (the IMU chains' branches 1 and 2 too, and _depth_imu's dropped frames: a header and the state, no rows).  The staged calls record
 * nothing.
 *   header (IMMESH_LIO_FEED_HDR int64): IMMESH_FEED_SCAN number; KIND (IMMESH_FEED_KIND_*); BRANCH (0 LiDAR-only, else the IMU
 *     chain's 1/2/3); ITERS run; MATCHES of the last IESKF iteration (m_effct_feat_num); CONVERGED flag of that iteration; ERR (the
 *     IM_LC_ERR flags); ROW_BEGIN, ROW_EFFECT_END, ROW_END: the scan's effect rows [BEGIN, EFFECT_END) and registered rows
 *     [EFFECT_END, END), numbered over the feed; SOURCE of the registered rows (0 none, 1 down-sampled, 2 full scan); ROWS_LOST.
 *   state: the 348 doubles the scan ended with, bit-identical to immesh_lio_wait right after it (branches 1 and 2: the state as the
 *     branch left it).
 *   rows: effect = 1: immesh_lio_effect_cloud right after the scan (row_index = its scan_index).  registered = 1:
 *     immesh_lio_registered_cloud(h, NULL, ..., point_skip); registered = 2: on _raw, _imu, _depth and _depth_imu, immesh_lio_registered_cloud of
 *     immesh_voxelgrid_input_points (stride 3, intensity column -1; _depth: its device count), on _raw_i and _imu_i immesh_lio_frontend_cloud(h, vg, 1,
 *     point_skip), elsewhere (no full scan) source 1.  row_index of a registered row: -1.
 *   A scan whose rows exceed max_rows keeps its header and state and sets ROWS_LOST.  A loss never fails a step or changes the state,
 *   the map or the mesh.
 * immesh_lio_feed(h, since_scan, wait, ...) returns the scans (since_scan, newest finished] oldest first, their states (or NULL) and
 *   their rows concatenated in scan order (or NULL).  wait = 0 never blocks on unfinished work; wait = 1 first waits for the newest
 *   queued scan.  counts = [scans, rows, newest finished, newest queued].  cap_scans = 0: a count query (IMMESH_OK, nothing written).
 *   More scans than cap_scans, or rows != NULL and more rows than cap_rows: IMMESH_E_CAPACITY with the counts, nothing written.  A
 *   scan of the range whose header or rows were overwritten in the rings: IMMESH_E_RANGE with counts[2] set (read on from there).
 *   since_scan < 0 or beyond the newest queued scan, the feed off, or a sharded handle: IMMESH_E_INVALID. */
typedef struct {
    int64_t max_scans;   /* header + state ring, in scans */
    int64_t max_rows;    /* row ring, rows of IMMESH_SCAN_PUB_COLS floats */
    int effect;          /* 1: record publish_effect_world's rows */
    int registered;      /* 0 none; 1 the down-sampled scan; 2 the full scan where the chain has one */
    int point_skip;      /* >= 1 */
    int pad;
} immesh_lio_feed_config;
#define IMMESH_LIO_FEED_HDR 12
#define IMMESH_FEED_SCAN 0
#define IMMESH_FEED_KIND 1
#define IMMESH_FEED_BRANCH 2
#define IMMESH_FEED_ITERS 3
#define IMMESH_FEED_MATCHES 4
#define IMMESH_FEED_CONVERGED 5
#define IMMESH_FEED_ERR 6
#define IMMESH_FEED_ROW_BEGIN 7
#define IMMESH_FEED_ROW_EFFECT_END 8
#define IMMESH_FEED_ROW_END 9
#define IMMESH_FEED_SOURCE 10
#define IMMESH_FEED_ROWS_LOST 11
/* IMMESH_FEED_KIND: the entry point that queued the scan */
#define IMMESH_FEED_KIND_STEP 0
#define IMMESH_FEED_KIND_STEP_DEV 1
#define IMMESH_FEED_KIND_STEP_ASYNC 2
#define IMMESH_FEED_KIND_STEP_ASYNC_DEV_N 3
#define IMMESH_FEED_KIND_RAW 4
#define IMMESH_FEED_KIND_RAW_I 5
#define IMMESH_FEED_KIND_IMU 6
#define IMMESH_FEED_KIND_IMU_I 7
#define IMMESH_FEED_KIND_DEPTH 8   /* immesh_lio_step_async_depth */
#define IMMESH_FEED_KIND_DEPTH_IMU 9   /* immesh_lio_step_async_depth_imu */
/* IMMESH_FEED_BRANCH of an immesh_lio_step_async_depth_imu frame that sync_packages dropped (a cloud of <= 1 point, or a carry overflow) */
#define IMMESH_FEED_BRANCH_DROPPED 4
int immesh_lio_feed_enable(immesh_lio_t* h, const immesh_lio_feed_config* cfg /* NULL: off */);
int immesh_lio_feed(immesh_lio_t* h, int64_t since_scan, int wait, int64_t* scans /*[cap_scans][12]*/, double* states /*[cap_scans][348] or NULL*/,
                    int cap_scans, float* rows /*[cap_rows][4] or NULL*/, int32_t* row_index /*[cap_rows] or NULL*/, int64_t cap_rows,
                    int64_t* counts /*[4]*/);
/* Plane-map markers in the scan feed: pubPlaneMap(m_feat_map, voxel_pub, state.pos_end), which the reference calls after
 * map_incremental_grow and after voxel_map_init when voxel/pub_plane_en is set (src/voxel_mapping.cpp:1975-1976, :1899-1900),
 * recorded on the device for each scan the feed records, behind the scan's map update and before the scan counts as finished.
 * immesh_lio_feed_markers_enable(h, max_rows): max_rows > 0 turns the recording on with a ring of max_rows rows of
 *   IMMESH_PLANE_MARKER_COLS doubles; 0 turns it off and frees the ring.  Drains h and drops its captured launch sequence.  Needs the
 *   feed on; every immesh_lio_feed_enable call (NULL included) turns the markers off.  max_rows outside [0, 2^32], the feed off,
 *   or a sharded handle: IMMESH_E_INVALID.  The recording keeps 16 bytes per root slot of device scratch for the key sort.
 * A scan's record equals what immesh_voxelmap_plane_markers would return if it were called right after that scan: the same rows in
 *   the same order, the same counters and roots walked, the same flags consumed and children held back.  The IMU chain's branch 2
 *   (voxel_map_init) walks as well; branch 1 records no rows and walks nothing.  The blocking call stays allowed: the rows it returns
 *   are consumed and never appear in the feed.  Staged calls record nothing, so the first message after immesh_voxelmap_build comes
 *   from one blocking call before the steps are queued.
 *   header (IMMESH_LIO_FEED_MARKER_HDR int64): IMMESH_MARKER_SCAN (the feed's scan number); ROW_BEGIN, ROW_END: the scan's rows,
 *     numbered over the marker ring; ROWS_NEEDED: the rows the walk counted; LOST; ROOTS_WALKED; PLANES, SUB_PLANES, SUB_SUB_PLANES,
 *     UPDATES: the reference's counters (immesh_voxelmap_plane_markers' counts[0..3]).
 *   A scan whose rows exceed max_rows sets LOST, writes no rows and consumes nothing: its roots stay pending and are published with a
 *   later scan, as if the node had skipped pubPlaneMap on that scan.  Size the ring from ROWS_NEEDED.  A loss never changes the
 *   state, the map or the mesh.
 * immesh_lio_feed_markers(h, since_scan, wait, ...): the marker records of the scans (since_scan, newest finished], oldest first, and
 *   their rows concatenated (rows may be NULL); since_scan, wait, counts, the count query, IMMESH_E_CAPACITY and IMMESH_E_RANGE as in
 *   immesh_lio_feed.  Scans queued before the markers were enabled have no record: a range that holds one gives IMMESH_E_RANGE.
 *   Never synchronises h's stream.  The markers off, the feed off, or a sharded handle: IMMESH_E_INVALID. */
#define IMMESH_LIO_FEED_MARKER_HDR 10
#define IMMESH_MARKER_SCAN 0
#define IMMESH_MARKER_ROW_BEGIN 1
#define IMMESH_MARKER_ROW_END 2
#define IMMESH_MARKER_ROWS_NEEDED 3
#define IMMESH_MARKER_LOST 4
#define IMMESH_MARKER_ROOTS_WALKED 5
#define IMMESH_MARKER_PLANES 6
#define IMMESH_MARKER_SUB_PLANES 7
#define IMMESH_MARKER_SUB_SUB_PLANES 8
#define IMMESH_MARKER_UPDATES 9
int immesh_lio_feed_markers_enable(immesh_lio_t* h, int64_t max_rows /* 0: off */);
int immesh_lio_feed_markers(immesh_lio_t* h, int64_t since_scan, int wait, int64_t* scans /*[cap_scans][10]*/, int cap_scans,
                            double* rows /*[cap_rows][16] or NULL*/, int64_t cap_rows, int64_t* counts /*[4]*/);
/* Host-side formatters of a recorded state (no device work).
 * immesh_odometry_pose: out = pos_end, then the quaternion x y z w that publish_odometry, publish_path and publish_mavros send:
 *   (roll, pitch, yaw) = RotMtoEuler(rot_end) (include/so3_math.h: sy = sqrt(r00^2 + r10^2); sy >= 1e-6: roll = atan2(r21, r22),
 *   pitch = atan2(-r20, sy), yaw = atan2(r10, r00); else roll = atan2(-r12, r11), pitch = atan2(-r20, sy), yaw = 0), then
 *   tf::createQuaternionMsgFromRollPitchYaw: with c_a = cos(a / 2), s_a = sin(a / 2) of a = roll r, pitch p, yaw y,
 *   x = s_r c_p c_y - c_r s_p s_y, y = c_r s_p c_y + s_r c_p s_y, z = c_r c_p s_y - s_r s_p c_y, w = c_r c_p c_y + s_r s_p s_y.
 *   This is not the quaternion of rot_end that Eigen would give (immesh_kitti_pose_line's).
 * immesh_lio_state_line: dump_lio_state_to_log's line (src/voxel_mapping_common.cpp:100-117): t, Log(rot_end) (include/so3_math.h:
 *   theta = 0 when the trace exceeds 3 - 1e-6, else acos((trace - 1) / 2); K = (r21 - r12, r02 - r20, r10 - r01); K / 2 when
 *   |theta| < 0.001, else theta / 2 / sin(theta) K), pos_end, three zeros, vel_end, three zeros, bias_g, bias_a, gravity, each
 *   printed "%lf ", then "\r\n".  t is the caller's (lidar_beg_time - first_lidar_time).  A line longer than cap - 1: IMMESH_E_CAPACITY. */
int immesh_odometry_pose(const double* state /*[>= 12]*/, double* out /*[7]*/);
int immesh_lio_state_line(const double* state /*[>= 24]*/, double t, char* buf, int cap);

/* device time (ms, CUDA events on the handle's stream) of the stages of the last immesh_lio_step call:
 * [0] whole step incl. H2D, [1] residual+solve iterations, [2] map update */
int immesh_lio_last_timing(immesh_lio_t* h, double* ms /*[3]*/);
/* work accounting of the last immesh_lio_step* call, used for the roofline arithmetic: [points in the scan, root voxels in the map,
 * plane refits (init_plane calls) of the map update, stored points those refits read] */
int immesh_lio_work_stats(immesh_lio_t* h, int64_t* out /*[4]*/);

/* ---- meshing handle: Global_map + Triangle_manager of the voxel-wise mesher ---------------------------- */
typedef struct immesh_mesh_config {
    double points_minimum_scale; /* meshing/points_minimum_scale * distance_scale -> m_minimum_pts_size */
    double voxel_resolution;     /* meshing/voxel_resolution * distance_scale -> m_voxel_resolution */
    int number_of_pts_append_to_map; /* appending_pts_frame (src/ImMesh_node.cpp:93-98) */
    int max_vertices;            /* capacities (0 = defaults) */
    int max_triangles;
    int max_voxels;
    int max_frame_points;
} immesh_mesh_config;

int immesh_mesh_create(const immesh_mesh_config* cfg, immesh_mesh_t** out);
int immesh_mesh_destroy(immesh_mesh_t* h);
/* incremental_mesh_reconstruction(frame_pts, pose_q, pose_t, frame_idx) (src/ImMesh_mesh_reconstruction.cpp:92-267):
 * append vertices, find activated voxels, per voxel retrieve + dilate + project + 2-D Delaunay + pull/commit,
 * then push.  world_xyz is the full-resolution scan already in the world frame (float, as pcl::PointXYZI). */
int immesh_mesh_push_frame(immesh_mesh_t* h, const float* world_xyz /*[n][3]*/, int n, const double* pose_t /*[3]*/, int frame_idx);
/* same, with the world-frame scan already resident in device memory */
int immesh_mesh_push_frame_dev(immesh_mesh_t* h, const float* d_world_xyz, int n, const double* pose_t, int frame_idx);
/* The hand-off at the end of Voxel_mapping::map_incremental_grow (src/ImMesh_mesh_reconstruction.cpp:413-417):
 * transformLidar of the full-resolution body-frame scan with the state the localization handle just converged to
 * (on the device, no host round trip of the world cloud), then incremental_mesh_reconstruction on it.
 * on_device != 0: body_xyz is a device pointer. */
int immesh_mesh_push_frame_from_lio(immesh_mesh_t* h, immesh_lio_t* lio, const float* body_xyz, int n, int on_device);
/* queued variant: the frame is transformed right behind the localization step that produced its pose (on the
 * localization stream) and meshed on the mesh stream while the next scan is being localised; immesh_mesh_wait drains. */
int immesh_mesh_push_frame_from_lio_async(immesh_mesh_t* h, immesh_lio_t* lio, const float* body_xyz, int n, int on_device);
int immesh_mesh_wait(immesh_mesh_t* h);
/* Depth-camera frames: one depth image unprojected on the device, inside the frame's own launch sequence, into the world-frame points
 * of an ordinary mesh frame -- the ImMesh paper's depth-image workload (AirSim 640 x 480 depth streams turned into point clouds, Table VI),
 * without a host pass over the pixels or a copy of the cloud.
 *   Sampling: pixel (u, v) is sampled iff u % stride == 0 and v % stride == 0; the valid samples become the frame's points in ascending
 *     pixel order (v major, u minor).  The image is width x height pixels with rows pitch_bytes apart (0: tight), float32 metres
 *     (IMMESH_DEPTH_F32) or uint16 counts of depth_scale metres (IMMESH_DEPTH_U16).
 *   Arithmetic, float64 in this order without FMA:
 *     d = raw (f32) or raw * depth_scale (u16); a u16 raw == 0 and a non-finite f32 raw are invalid;
 *     a = (u - cx) / fx, b = (v - cy) / fy;
 *     z = d (IMMESH_DEPTH_PLANAR: depth along the optical axis, AirSim DepthPlanar) or
 *     z = d / sqrt((a*a + b*b) + 1) (IMMESH_DEPTH_RANGE: distance along the ray, AirSim DepthPerspective);
 *     x = a * z, y = b * z; the pixel is valid iff z_min <= z <= z_max;
 *     w_i = (float)(((R[i][0]*x + R[i][1]*y) + R[i][2]*z) + t[i]) with R = cam_R (row-major), t = cam_t.
 *   Axes: cam_R / cam_t map the camera frame to the world, with OpenCV axes (x right, y down, z forward).  A caller whose pose uses
 *     the OpenGL convention (y up, z backward) multiplies its rotation on the right by diag(1, -1, -1) first.
 *   The frame is then immesh_mesh_push_frame of those points at pose_t = cam_t (the camera centre is the sensor position of
 *     correct_triangle_index): its point count, append_point_step and candidate count are set on the device from the valid count, with
 *     the rule of immesh_mesh_push_frame.  The change feed, the frame feed (KIND = IMMESH_MFEED_KIND_DEPTH; N_POINTS and STEP are the
 *     device values), the reinforcement and the queued view follow it as any frame.
 * immesh_mesh_push_depth(h, f, depth, on_device): blocking, as immesh_mesh_push_frame.  on_device != 0: depth is a device pointer, read
 *   in place.  A host image is staged, sampled pixels only, through the handle's pinned slots.
 * immesh_mesh_push_depth_async: queued (graph-replayed, no host synchronisation); immesh_mesh_wait drains it and returns its status.
 *   A device image must stay unchanged until the frame has run.
 * immesh_mesh_depth_points(h, xyz, cap, n): blocking; the newest depth frame's world points, *n of them.  cap = 0: a count query;
 *   *n > cap: IMMESH_E_CAPACITY (nothing written).  No depth frame pushed yet: IMMESH_E_INVALID.
 * Errors: IMMESH_E_INVALID for a null or misaligned image, fx or fy zero or non-finite, cx, cy, cam_R or cam_t non-finite, width or
 *   height < 1, a pitch below the row's bytes or not a multiple of the pixel size, stride < 1, an unknown format or kind,
 *   !(0 <= z_min < z_max < inf), a u16 depth_scale that is not positive and finite, or a sharded handle; IMMESH_E_CAPACITY when the
 *   sampled pixels exceed max_frame_points; otherwise the codes of immesh_mesh_push_frame (e.g. IMMESH_E_RANGE far from cam_t). */
#define IMMESH_DEPTH_F32 0
#define IMMESH_DEPTH_U16 1
#define IMMESH_DEPTH_PLANAR 0
#define IMMESH_DEPTH_RANGE 1
typedef struct immesh_depth_frame {
    int width, height;
    int64_t pitch_bytes;  /* bytes between rows; 0 = width * bytes per pixel */
    int format;           /* IMMESH_DEPTH_F32 or IMMESH_DEPTH_U16 */
    int kind;             /* IMMESH_DEPTH_PLANAR or IMMESH_DEPTH_RANGE */
    double depth_scale;   /* metres per u16 count (ignored for f32) */
    double fx, fy, cx, cy;
    double z_min, z_max;  /* valid z range, metres: 0 <= z_min < z_max < inf */
    int stride;           /* >= 1: every stride-th pixel of every stride-th row */
    int pad;
    double cam_R[9];      /* camera to world, row-major, OpenCV camera axes */
    double cam_t[3];      /* camera centre in the world */
} immesh_depth_frame;
int immesh_mesh_push_depth(immesh_mesh_t* h, const immesh_depth_frame* f, const void* depth, int on_device);
int immesh_mesh_push_depth_async(immesh_mesh_t* h, const immesh_depth_frame* f, const void* depth, int on_device);
int immesh_mesh_depth_points(immesh_mesh_t* h, float* xyz /*[cap][3]*/, int cap, int* n);
/* host time (ms) the queueing calls spent blocked on a busy staging slot (back-pressure from the device, not work) since the
 * last call: out[0] localization handle, out[1] meshing handle; either handle may be NULL */
int immesh_host_wait_ms(immesh_lio_t* lio, immesh_mesh_t* h, double* out /*[2]*/);
/* CUDA-event time (ms) of everything queued on both handles between the two marks */
int immesh_pipeline_mark_begin(immesh_lio_t* lio);
int immesh_pipeline_mark_end(immesh_lio_t* lio, immesh_mesh_t* h, double* ms);
/* counts: [n_vertices, n_live_triangles, frame_new_vertices, frame_voxels_meshed, frame_added, frame_removed, n_voxels, n_activated] */
int immesh_mesh_counts(immesh_mesh_t* h, int64_t* out /*[8]*/);
/* Long runs: the same three calls as immesh_lio_capacity / _reserve / _set_growth for the mesh handle's pools -- vertices (with the
 * xi-grid and the vertex chunks), triangles (with the triple hash) and mesh voxels (max_voxels, with the voxel hash).  capacity:
 * out = [vertex capacity, vertices, triangle capacity, triangles allocated, voxel capacity, voxels, device bytes, growths].  The
 * automatic check runs before every immesh_mesh_push_frame* call and before a batched frame (not inside one).  The per-frame capacities
 * (max_frame_points and the frame's work and list capacities) do not grow.  A grown handle computes what a handle created at the
 * larger capacities computes. */
int immesh_mesh_capacity(immesh_mesh_t* h, int64_t* out /*[8]*/);
int immesh_mesh_reserve(immesh_mesh_t* h, int64_t vertices, int64_t triangles, int64_t voxels);
int immesh_mesh_set_growth(immesh_mesh_t* h, int64_t max_bytes);
/* Triangle_manager::get_all_triangle_list (src/meshing/r3live/triangle.cpp:12-33) + the vertex array:
 * live triangles as ascending sorted (i<j<k) id triples with their m_index_flip. */
int immesh_mesh_snapshot(immesh_mesh_t* h, float* vertices /*[nv][3] or NULL*/, int32_t* triangles /*[nt][3] or NULL*/,
                         int32_t* flips /*[nt] or NULL*/);
/* save_to_ply_file (src/meshing/mesh_rec_geometry.cpp:71-131, smooth_factor == 0): binary little-endian PLY of a snapshot -- float x y z
 * per vertex, one face per triangle oriented by the reference's rule (m_index_flip != 0: p0 p1 p2, else p0 p2 p1).  Host-side only. */
int immesh_write_ply(const char* path, const float* vertices /*[nv][3]*/, int nv, const int32_t* triangles /*[nt][3]*/,
                     const int32_t* flips /*[nt] or NULL*/, int nt);
/* pcl::io::savePCDFileBinary of the vertex cloud, written by save_to_ply_file next to the PLY (mesh_rec_geometry.cpp:129).  Host-side only. */
int immesh_write_pcd(const char* path, const float* vertices /*[nv][3]*/, int nv);
/* smooth_all_pts(smooth_factor, knn) (src/meshing/mesh_rec_geometry.cpp:60-69) = Global_map::smooth_pts on every vertex
 * (src/meshing/r3live/pointcloud_rgbd.cpp:932-958, maximum_smooth_dis = g_kd_tree_accept_pt_dis = 1.25 * voxel_resolution): exact knn on the
 * device, neighbours 1..knn-1 closer than the limit averaged, smoothed = p (1 - f) + mean f.  Updates the vertices' smoothed positions
 * (set_smooth_pos) and returns them (smoothed may be NULL); save_to_ply_file with smooth_factor != 0 writes exactly these positions. */
int immesh_mesh_smooth_all(immesh_mesh_t* h, double smooth_factor, int knn /*<= 32*/, double* smoothed /*[n_vertices][3] or NULL*/);
/* Region-bucketed triangle stream of the viewer (Triangle_manager::insert_triangle_to_list, src/meshing/r3live/triangle.cpp:35-53): every live
 * triangle belongs to region round(centre / region_size).  Output: regions in ascending key order (region_keys [nr][3], region_offsets
 * [nr + 1] into `triangles`), triangles [n_live][3] grouped by region, ascending triples inside a region. */
int immesh_mesh_region_stream(immesh_mesh_t* h, double region_size, int32_t* region_keys /*[cap][3] or NULL*/, int32_t* region_offsets /*[cap+1] or NULL*/,
                              int cap_regions, int32_t* triangles /*[n_live][3] or NULL*/, int* n_regions);
/* The mesh viewer's triangle buffers: synchronize_triangle_list_for_disp (src/meshing/mesh_rec_display.cpp:220-258, every 100 ms from
 * service_refresh_and_synchronize_triangle :262-271) -> unparse_triangle_set_to_vector (:78-104) + get_axis_min_max (:105-137) over the
 * region sets of Triangle_manager::insert_triangle_to_list (src/meshing/r3live/triangle.cpp:35-53).
 *   Regions: a triangle's region is the key of immesh_mesh_region_stream.  keys == NULL: every non-empty region, ascending key order;
 *     else exactly the n_keys regions listed, in the caller's order, an empty segment for a region without triangles (a key outside
 *     the mesh's key range holds none); a repeated key is IMMESH_E_INVALID.  Inside a region, ascending (i<j<k) triples.
 *     region_keys [n_regions][3] and region_offsets [n_regions + 1] (into the rows) describe the segments.
 *   Lazy smoothing: before any row is written, every vertex of an emitted triangle whose m_smoothed flag is clear is smoothed as
 *     Global_map::smooth_pts (src/meshing/r3live/pointcloud_rgbd.cpp:932-958) does it: its knn nearest vertices (ties to the lower id,
 *     the immesh_knn rule), neighbours 1..knn-1 closer than g_kd_tree_accept_pt_dis = 1.25 voxel_resolution averaged from their RAW
 *     positions, p (1 - f) + mean f (no neighbour inside the limit: the reference's division by zero, NaN); the result is stored as
 *     the vertex's smoothed position and the flag is set (set_smooth_pos).  Only vertices of the selected regions are touched.
 *     The flag is set by the mesher's dilation (retrieve_neighbor_pts_kdtree, src/meshing/mesh_rec_geometry.cpp:336-377), by
 *     immesh_mesh_smooth_all and by this call; a vertex is appended with it clear.  *n_smoothed (or NULL): vertices smoothed here.
 *     The viewer uses g_ply_smooth_factor = 1.0 and g_ply_smooth_k = 20.
 *   Rows: tri_xyz [n_tris][9] = (float) of the three vertices' smoothed positions, ascending ids (get_pos(1).cast<float>()); tri_ids
 *     [n_tris][3] the triples.  Either may be NULL.
 *   axis_min_max [6] (min xyz, max xyz; or NULL) is read and updated over the emitted floats with the reference's strict < / >
 *     comparisons, in row order; start it at +-1e8 as :264 does.
 *   *n_tris > cap or *n_regions > cap_regions: IMMESH_E_CAPACITY with the counts needed; nothing is written and nothing is smoothed
 *     (cap = 0: a pure count query).  region_size <= 0 or knn outside [1, 32]: IMMESH_E_INVALID.  A region key outside the mesh's
 *     key range (+-1048000): IMMESH_E_RANGE.
 *   Blocking: waits for the work queued on h, the frames of immesh_mesh_push_frame_from_lio_async included.  The smoothed positions
 *     stored here are the ones later frames' correct_triangle_index (mesh_rec_geometry.cpp:399-433) reads -- in the reference a race
 *     with the viewer thread, here ordered between frames.
 *   A sharded handle: every replica holds the same triangle store, smoothed positions and flags, so every rank returns the same rows
 *     and applies the same write-back, without an exchange. */
#define IMMESH_REGION_TRI_FLOATS 9
int immesh_mesh_region_buffers(immesh_mesh_t* h, double region_size, const int32_t* keys /*[n_keys][3] or NULL*/, int n_keys,
                               double smooth_factor, int knn /*[1,32]*/,
                               float* tri_xyz /*[cap][9] or NULL*/, int32_t* tri_ids /*[cap][3] or NULL*/, int cap,
                               int32_t* region_keys /*[cap_regions][3] or NULL*/, int32_t* region_offsets /*[cap_regions+1] or NULL*/,
                               int cap_regions, float* axis_min_max /*[6] in/out or NULL*/,
                               int* n_regions, int* n_tris, int* n_smoothed /*or NULL*/);
/* reconstruct_mesh_from_pointcloud(frame_pts, minimum_pts_distance) (src/ImMesh_mesh_reconstruction.cpp:328-345; the offline whole-cloud
 * entry of config/offline_pointcloud.yaml): VoxelGrid down-sampling with leaf = minimum_pts_distance, then one
 * incremental_mesh_reconstruction frame with the identity pose.  xyz: [n][3] host array, or device pointer with on_device = 1. */
int immesh_mesh_reconstruct_from_pointcloud(immesh_mesh_t* h, immesh_voxelgrid_t* vg, const float* xyz, int n, int on_device, double minimum_pts_distance,
                                            int* n_downsampled /*or NULL*/);
/* One incremental_mesh_reconstruction frame (src/ImMesh_mesh_reconstruction.cpp:92-267) of any size, executed in bounded batches.
 *   The append (append_points_to_global_map, src/meshing/r3live/pointcloud_rgbd.cpp:411-552, append_point_step = max(1, round(n /
 *     appending_pts_frame)) with the integer division in 64 bits) runs in chunks of <= batch_points candidates, in scan order; the
 *     activation test (:132-151) runs once after the last chunk; the meshed voxels are then processed in batches of <= batch_voxels:
 *     first every batch's dilation with its smoothing (retrieve_neighbor_pts_kdtree), then every batch's triangulation, pull and commit
 *     against the store as it was before the frame, its new facets pushed at once; removals are applied after the last batch.
 *   Result: bit-identical to one unbatched frame on the same points (vertices and ids, smoothed positions and m_smoothed flags, facets,
 *     m_index_flip, immesh_mesh_counts), whatever the batch sizes.  The orientation priority is the voxel's rank among the frame's meshed
 *     voxels in (x, y, z) key order, so, unlike immesh_mesh_push_frame, no voxel is too far from pose_t (IMMESH_E_RANGE).
 *   batch_points: <= max_frame_points, 0 = max_frame_points.  batch_voxels: <= the frame's work capacity (max_voxels / 16 clamped to
 *     [65536, 262144], or max_voxels when smaller), 0 = that capacity.  Other values, or a sharded handle: IMMESH_E_INVALID.  A batch whose
 *     facets or dilated sets overflow the per-frame lists returns IMMESH_E_CAPACITY (flag LIST_CAP): use smaller batches.
 *   world_xyz: [n][3] host array, read chunk by chunk through the handle's pinned slots (double-buffered, not copied whole), or a
 *     device pointer with on_device = 1.  Scratch beyond the mesh pools is allocated by the first call and sized by the handle's
 *     capacities only.  stats (or NULL): [append chunks, voxel batches, scratch bytes, facet add entries].  Blocking; frames queued
 *     before the call are drained first. */
int immesh_mesh_push_frame_batched(immesh_mesh_t* h, const float* world_xyz /*[n][3]*/, int64_t n, int on_device, const double* pose_t /*[3]*/,
                                   int batch_points, int batch_voxels, int64_t* stats /*[4] or NULL*/);
/* reconstruct_mesh_from_pointcloud (src/ImMesh_mesh_reconstruction.cpp:328-345) on a cloud of any size.  PCL's VoxelGrid decision is
 * made on the whole cloud (its bounding box reduced chunk by chunk with the VoxelGrid's own kernels, so "leaf size too small" matches
 * immesh_voxelgrid_filter exactly).  Passed through (the usual case at minimum_pts_distance = 0.01 m for clouds wider than about 13 m):
 * the raw cloud goes into the batched frame and vg's capacity does not matter.  Filtered: vg down-samples it (more than vg's max_points:
 * IMMESH_E_CAPACITY) and the result goes into the batched frame.  Identity pose.  *n_meshed_points: points given to the frame. */
int immesh_mesh_reconstruct_from_pointcloud_batched(immesh_mesh_t* h, immesh_voxelgrid_t* vg, const float* xyz, int64_t n, int on_device,
                                                    double minimum_pts_distance, int batch_points, int batch_voxels,
                                                    int64_t* n_meshed_points /*or NULL*/);
/* Depth rasterisation of the live mesh from a camera -- the reference's "LiDAR point-cloud reinforcement" (src/ImMesh_node.cpp:305-329:
 * draw_triangle into the depth camera, Cam_view::read_depth, convert_depth_buffer_to_truth_depth + unproject_point,
 * src/tools/openGL_libs/openGL_camera_view.cpp:316-418) as a CUDA rasteriser over the device-resident triangle store.
 *   intrinsics = fx, fy, cx, cy;  cam_R (row-major) / cam_t = m_camera_rot / m_camera_pos of Cam_view (world = R diag(1,-1,-1) p_cam + t)
 *   depth  [height][width]: metric depth along the optical axis of the nearest surface, -1 where none is closer than 0.99 z_far
 *   points [n][3] (+ point_pixel [n] = y * width + x): unproject_point of every valid pixel, ascending pixel order; may be NULL
 * Sampling rule (defined here; the reference leaves it to the GL implementation): samples at integer pixel coordinates, covered when
 * the three edge functions share a sign, 1/z interpolated affinely, triangles with a vertex outside (z_near, z_far) skipped. */
int immesh_mesh_render_depth(immesh_mesh_t* h, const double* intrinsics /*[4]*/, int width, int height, double z_near, double z_far,
                             const double* cam_R /*[9]*/, const double* cam_t /*[3]*/, float* depth, float* points, int32_t* point_pixel, int* n_points);
/* The LiDAR point-cloud reinforcement with the depth camera bound to the sensor (src/ImMesh_node.cpp:302-329, g_if_draw_depth with
 * g_if_depth_bind_cam), queued behind every mesh frame.  Per frame the reference takes the camera pose from the last meshed frames
 * (get_last_avr_pose, :169-206), rasterises the live mesh into the depth camera (draw_triangle, Cam_view::read_depth) and unprojects
 * every valid pixel (convert_depth_buffer_to_truth_depth + unproject_point, src/tools/openGL_libs/openGL_camera_view.cpp:316-418); the
 * points are drawn beside the current scan (display_reinforced_LiDAR_pts, src/meshing/mesh_rec_display.cpp:178-196).
 *   immesh_mesh_reinforce_enable: allocates the buffers once for the image and from then on every frame of immesh_mesh_push_frame,
 *     _dev, _from_lio, _from_lio_async (and reconstruct_from_pointcloud) queues, on the mesh stream right behind the frame and inside
 *     its captured graph, the camera pose, the depth image of the mesh as the frame left it and its points -- no host
 *     synchronisation, no allocation.  The batched frames (push_frame_batched) are not followed.  intrinsics = NULL turns it off and
 *     frees the buffers.  Either call drains the frames in flight.  Bad intrinsics (non-finite, fx or fy = 0), image size outside
 *     [1, 2^26] pixels, z range not 0 < z_near < z_far < inf, win outside [1, 63], or a sharded handle: IMMESH_E_INVALID.
 *   The reference's camera (ImMesh_node.cpp:285-293): 640 x 480, m_camera_focus = 400, the z range of the GL camera (z_near 0.1,
 *     z_far 1500), win_ssd = 1.  Cam_view::set_gl_projection (openGL_camera_view.cpp:83-101) rounds the width up to a multiple of 4
 *     and sets m_camera_intrinsic = [focus 0 w/2; 0 focus h/2; 0 0 1] with integer halves: intrinsics = (focus, focus, w / 2, h / 2),
 *     (400, 400, 320, 240) for the defaults.
 *   Camera pose of frame n (the handle's frames counted from 1; the reference's current frame is n - 1): the frames
 *     [max(1, n - win), n) that were handed over by the localization handle (they recorded rot_end, pos_end of the pose they were
 *     transformed with) give q_first exp(mean_i log(q_first^-1 q_i)) * lidar_frame_to_camera_frame = [0 0 -1; -1 0 0; 0 1 0] (quaternions
 *     from the rotation matrices as Eigen::Quaterniond does it, Sophus SO3 log / exp) and the mean position; the result is
 *     m_camera_rot / m_camera_pos as in immesh_mesh_render_depth.  The first frame (the reference's cur < 1) gets the identity pose;
 *     so does a window holding no frame with a pose (world-frame frames carry none; the reference divides by zero there).
 *   immesh_mesh_reinforce_pose(h, cam_R, cam_t): the caller's camera pose instead, from the next queued frame on, for every frame
 *     (the form for frames pushed with world points); NULL, NULL returns to the sensor-bound pose.  Enabling starts sensor-bound.
 *   Result: exactly immesh_mesh_render_depth at that pose -- both run the same tiled rasteriser (16 x 16 pixel tiles; the triangles
 *     binned by their pixel boxes), so the same depth image bit for bit and the same points and pixels in ascending pixel order.
 *   immesh_mesh_reinforced_cloud: blocking read of the newest queued frame's result (waits for that frame only).  The result is
 *     double-buffered: a frame queued after the read started writes the other buffer.  depth [height][width] (-1 where empty),
 *     points [n][3], point_pixel [n] (y * width + x), pose_out [12] = R row-major, t; each may be NULL.  *n_out > cap:
 *     IMMESH_E_CAPACITY with *n_out = points needed, nothing written (cap = 0: a count query).  Not enabled, no frame queued since
 *     enable, or a sharded handle: IMMESH_E_INVALID. */
int immesh_mesh_reinforce_enable(immesh_mesh_t* h, const double* intrinsics /*[4] or NULL*/, int width, int height, double z_near, double z_far, int win);
int immesh_mesh_reinforce_pose(immesh_mesh_t* h, const double* cam_R /*[9] or NULL*/, const double* cam_t /*[3] or NULL*/);
int immesh_mesh_reinforced_cloud(immesh_mesh_t* h, float* depth /*[h][w] or NULL*/, float* points /*[cap][3] or NULL*/, int32_t* point_pixel /*[cap] or NULL*/,
                                 int cap, int* n_out, double* pose_out /*[12] or NULL*/);
/* The mesh viewer's shaded image, rendered on the device: the reference's draw_triangle (src/meshing/mesh_rec_display.cpp:273-282)
 * with the facet shader in face mode (g_display_face, if_light = true; src/shader/triangle_facets.vs / .fs), for a node without a
 * display.  A blocking call at the caller's camera, or an image queued behind every frame.  The view reads the mesh and writes nothing
 * on the handle (no vertex, m_smoothed flag, smoothed position, counter or change-feed row); it never smooths.
 *   style (NULL: positions 0, white):
 *     positions 0: the raw vertex positions (immesh_mesh_snapshot's); 1: the stored smoothed position (as float) where the vertex's
 *       m_smoothed flag is set, the raw position where it is not.  This draws what the viewer shows once its lazy smoothing has run:
 *       to match the viewer exactly, call immesh_mesh_region_buffers or immesh_mesh_smooth_all first.
 *     color_by_height 0: white (g_mesh_if_color = false, the viewer's default); 1: the height colour (set_color_by_axis on z).
 *     z_range: the height colour's range; both NaN: min / max z over the vertices of the live triangles, in the chosen positions, at
 *       render time.  Read only with color_by_height = 1; then ends that are not finite (other than both NaN) or z_range[0] >=
 *       z_range[1]: IMMESH_E_INVALID.
 *   Image rule (defined here, where GL leaves it to the implementation):
 *     Visibility: immesh_mesh_render_depth's sampling rule unchanged, with the positions of style.positions: samples at integer pixel
 *       coordinates, covered when the three edge functions share a sign (zero included), 1/z interpolated affinely, a triangle with a
 *       vertex outside (z_near, z_far) skipped.  At each pixel the nearest sample wins (the smaller bits of its float depth); on equal
 *       bits the lower (a, b, c) triple of vertex ids, so shared edges are drawn the same whatever the slot or bin order.
 *     depth [height][width] (may be NULL): what immesh_mesh_render_depth writes -- the metric depth, -1 at or beyond 0.99 z_far or
 *       where nothing was drawn; with positions 0 equal to immesh_mesh_render_depth's image bit for bit.
 *     rgba [height][width][4]: the winning triangle's vertices p0 p1 p2 in stored (ascending id) order, in float64 from the float
 *       positions, evaluated in the order written here without fused multiply-adds:
 *         normal n = (p1 - p0) x (p2 - p0); weights w_i = e_i (1 / z_i) from the sample's edge functions e_i;
 *         frag = ((w0 p0 + w1 p1) + w2 p2) / ((w0 + w1) + w2), the vertex colours interpolated with the same weights;
 *         light at the camera position: l = cam_t - frag;  d = n / |n| . l / |l| (components summed (x + y) + z, |v| likewise);
 *         per channel c = (0.2 + 0.5 |d|) colour;  byte = floor(clamp(c, 0, 1) 255 + 0.5) (NaN: 0);  alpha 255.
 *       Every pixel with a sample is shaded (also one whose depth is -1 beyond 0.99 z_far); a pixel without one is opaque black
 *       (0, 0, 0, 255), the reference's clear colour.
 *     Height colour of a vertex at z: t = (z - lo) / (hi - lo) in float32 with lo, hi the range as floats (t = 0 when hi == lo, as for
 *       a flat mesh); s = 1 - t clamped to [0, 1]; on the five stops blue (0,0,1), cyan (0,1,1), green (0,1,0), yellow (1,1,0), red
 *       (1,0,0) at a = 4 s: the stops floor(a) and ceil(a) mixed (1 - f) c0 + f c1 with f = a - floor(a), in float64; each channel
 *       truncated to the byte (unsigned char)(c 255); the vertex colour is byte / 255.  White is (1, 1, 1).
 *   immesh_mesh_render_view: blocking, at the caller's camera (the convention and argument checks of immesh_mesh_render_depth); bad
 *     style or a sharded handle: IMMESH_E_INVALID.
 *   immesh_mesh_view_enable: allocates the buffers once and from then on queues the image behind every frame of
 *     immesh_mesh_push_frame, _dev, _from_lio, _from_lio_async (and reconstruct_from_pointcloud), on the mesh stream after the
 *     reinforcement and inside the captured graph: no host synchronisation, no allocation.  The batched frames are not followed.
 *     intrinsics = NULL turns it off and frees the buffers; either call drains the frames in flight and drops the captured graph.
 *     Arguments as immesh_mesh_reinforce_enable's (bad ones: IMMESH_E_INVALID); enabling starts with the sensor-bound pose.  While the
 *     view is off, no launch, graph or output changes.  immesh_mesh_shard refuses a handle with the view on.
 *   immesh_mesh_view_pose(h, cam_R, cam_t, follow), from the next queued frame on:
 *     NULL, NULL (follow 0): the sensor-bound pose, the reinforcement's camera over `win` frames (the depth-view window with
 *       g_if_depth_bind_cam, ImMesh_node.cpp:312-319);
 *     follow 0: the fixed camera (cam_R, cam_t);
 *     follow 1: the follow camera (g_follow_cam, ImMesh_node.cpp:434-440): rotation cam_R, position the window's mean translation of
 *       the sensor-bound pose plus cam_t (a window without a pose contributes a zero translation).
 *     Not enabled, mismatched NULLs, follow not 0 / 1, follow 1 without a pose: IMMESH_E_INVALID.
 *   immesh_mesh_view_image: blocking read of the newest queued frame's image (waits for that frame only), double-buffered by
 *     frame & 1: rgba [h][w][4], depth [h][w], pose_out [12] = the frame's camera R row-major and t, frame_out = its frame number;
 *     each may be NULL.  Not enabled, no frame queued since enable, or a sharded handle: IMMESH_E_INVALID. */
typedef struct {
    int positions;        /* 0: raw vertex positions; 1: the smoothed position where m_smoothed is set, else the raw one */
    int color_by_height;  /* 0: white; 1: the height colour on z */
    double z_range[2];    /* height colour range; both NaN: min / max z over the live triangles' vertices at render time */
} immesh_view_style;
int immesh_mesh_render_view(immesh_mesh_t* h, const double* intrinsics /*[4]*/, int width, int height, double z_near, double z_far,
                            const double* cam_R /*[9]*/, const double* cam_t /*[3]*/, const immesh_view_style* style /*or NULL*/,
                            uint8_t* rgba /*[h][w][4]*/, float* depth /*[h][w] or NULL*/);
int immesh_mesh_view_enable(immesh_mesh_t* h, const double* intrinsics /*[4] or NULL*/, int width, int height, double z_near, double z_far, int win,
                            const immesh_view_style* style /*or NULL*/);
int immesh_mesh_view_pose(immesh_mesh_t* h, const double* cam_R /*[9] or NULL*/, const double* cam_t /*[3] or NULL*/, int follow);
int immesh_mesh_view_image(immesh_mesh_t* h, uint8_t* rgba /*[h][w][4] or NULL*/, float* depth /*[h][w] or NULL*/, double* pose_out /*[12] or NULL*/,
                           int64_t* frame_out /*or NULL*/);
/* The rest of the viewer's window in the queued view (src/ImMesh_node.cpp:422-470): the current scan (display_current_LiDAR_pts),
 * the reinforced points (display_reinforced_LiDAR_pts), the axis (g_axis_shader), the ground grid (g_ground_plane_shader), the
 * wireframe in place of the faces (draw_triangle with g_display_face = 0), the sensor's camera frustum (draw_camera_pose) and the
 * trajectory (draw_camera_trajectory).
 *   immesh_mesh_view_overlay(h, o): from the next queued frame on; needs the view enabled (immesh_mesh_view_enable, which, like
 *     disabling, clears the overlay).  Drains the frames in flight, drops the captured graph and allocates the overlay's buffers
 *     (per-pixel keys, trajectory ring, frustum) here and nowhere else.  o = NULL, or every layer off: no overlay; then no launch, graph
 *     or output differs from a handle that never called it.  Sizes or widths outside [0, 64], wireframe or axis_and_grid not 0 / 1,
 *     a non-finite or negative camera_size, path_capacity outside [1, 2^24] with path_width > 0, scan points with max_frame_points >=
 *     2^29, the view not enabled, or a sharded handle: IMMESH_E_INVALID.  The blocking immesh_mesh_render_view draws no overlay.
 *   Image rule (adds to immesh_mesh_render_view's, which stays as it is for the faces):
 *     Camera: the queued view's, in every mode.  Mesh vertices at style.positions.  Overlays unlit and opaque; their bytes by
 *       floor(clamp(c) 255 + 0.5): scan points, frustum and trajectory white; reinforced points magenta (255, 0, 255); the x, y, z axes
 *       red, green, blue; the grid grey 0.45 (115).
 *     Points: camera z in (z_near, z_far), depth the camera z as float; a point of size s at (u, v) covers the integer pixels with
 *       u - s/2 <= x < u + s/2 and v - s/2 <= y < v + s/2, cut to the image.
 *     Segments: the ends in camera space (float64), clipped to [z_near, z_far] (an end beyond a plane moves along the segment to it:
 *       s = (zp - za) / (zb - za), a + s (b - a), near first, then far; a segment wholly outside is dropped), then projected.  A line of
 *       width w, non-antialiased: x-major when |du| >= |dv|; it covers every integer column min(u0, u1) <= x < max(u0, u1), with
 *       t = (x - u0) / (u1 - u0) and v = v0 + t (v1 - v0) the rows v - w/2 <= y < v + w/2; 1/z = 1/z0 + t (1/z1 - 1/z0), the
 *       depth its float inverse.  A y-major line swaps the axes.  Float64 without fused multiply-adds.
 *     Wireframe: the edges (a, b), (b, c), (a, c) of each live triangle whose three vertices lie in (z_near, z_far), each from its
 *       lower vertex id to its higher, width 1, in the vertex colours of style (white or the height colour): w0 = (1 - t) / z0,
 *       w1 = t / z1, c = (w0 c0 + w1 c1) / (w0 + w1).  A shared edge rasterises to the same pixels from either triangle.
 *     Layers: the axis (from the origin, 1 m, width 10) and the grid (21 + 21 lines at z = 0, 10 m apart from -100 m to 100 m, line
 *       2i at x = 10 (i - 10) from y = -100 to 100 and line 2i + 1 at y = 10 (i - 10) from x = -100 to 100, width 1) with
 *       axis_and_grid; the scan: frame n's own world points for n >= 2 (frames counted from 1); the reinforced points: the queued
 *       reinforcement's cloud of the same frame, while the reinforcement is on; the frustum: frame n's rot_end R and pos_end t in
 *       float64 (a world-frame push carries no rotation: none), the 11-vertex strip of the hard-coded K (704.504153913163,
 *       703.6790228113778, 708.8501128392297, 562.7041625276061) and 1440 x 1080 at scale 1.5: fu = 1 / fx, u0 = -cx / fx (v
 *       likewise), xl = 1.5 u0, xh = 1.5 (1440 fu + u0), yl = 1.5 v0, yh = 1.5 (1080 fv + v0), the local vertices (xl,yl,1.5)
 *       (xh,yl,1.5) (xh,yh,1.5) (xl,yh,1.5) (xl,yl,1.5) 0 (xh,yl,1.5) 0 (xl,yh,1.5) 0 (xh,yh,1.5), in the world t_k + camera_size
 *       ((-R_k1 x + -R_k2 y) + R_k0 z), width 5; the trajectory: a line strip through the positions of the frames queued since this
 *       call (a localization frame's pos_end, a world-frame push's pose_t), the newest path_capacity kept, oldest first.
 *     Visibility: per pixel the smallest float depth bits win; on equal bits the earlier layer in the reference's draw order (scan,
 *       reinforced, axis, grid, mesh, frustum, trajectory), inside a layer the lower index (point order; segment order as listed; for
 *       faces the lower triple; for edges the lower (triple, edge)).
 *     depth of immesh_mesh_view_image: unchanged, the faces' depth image, also with the wireframe.  Batched frames are not followed. */
typedef struct {
    int    wireframe;              /* 1: the live triangles' edges instead of the faces (g_display_face = 0) */
    int    scan_point_size;        /* pixels; 0: off.  Reference 2 */
    int    reinforced_point_size;  /* pixels; 0: off.  Reference 2.  Drawn only while the reinforcement is enabled */
    int    axis_and_grid;          /* g_if_draw_z_plane (reference: on) */
    double camera_size;            /* g_display_camera_size; 0: no frustum.  Reference 1.0 */
    int    path_width;             /* g_draw_path_size + 2; 0: no trajectory.  Reference 4 */
    int    path_capacity;          /* positions kept for the trajectory; the oldest drop out */
} immesh_view_overlay;
int immesh_mesh_view_overlay(immesh_mesh_t* h, const immesh_view_overlay* o /* NULL: none */);
/* The change feed: each frame's added and removed triangles (the reference's per-frame added_triangle_list / removed_triangle_list,
 * src/ImMesh_mesh_reconstruction.cpp:122-123, 209-244), recorded on the device, so that a caller that keeps its own copy of the mesh
 * (publisher, remote viewer, recorder) applies the difference instead of calling immesh_mesh_snapshot after every frame.
 *   The state described is what immesh_mesh_snapshot returns: the vertices (raw x y z, ids in append order) and the live triangles
 *     as ascending (i<j<k) triples with their m_index_flip.  Frame f (the handle's frames counted from 1; a batched frame is one frame)
 *     appended the vertex ids [v_begin, v_end) and has one row (a, b, c, code) per triangle whose (live, flip) state differs between
 *     the end of frame f - 1 and the end of frame f: code 0 removed; 2 | flip made live; 4 | flip stayed live with its flip changed
 *     (an "existing" facet re-oriented by correct_triangle_index, src/meshing/mesh_rec_geometry.cpp:399-433).  The rows are the net
 *     difference (a triangle touched without a change of state gives none), in ascending (a, b, c) order inside a frame: the same with
 *     and without CUDA graphs and for any batch sizes.  Applying them to immesh_mesh_snapshot's result at frame f - 1 gives its
 *     result at frame f bit for bit.
 *   immesh_mesh_changes_enable(h, max_rows, max_frames): drains the frames in flight, allocates the feed (a ring of max_rows rows, the
 *     headers of the last max_frames frames, a per-frame list of min(max_rows, 2^21) touched triangles, a byte and a stamp per
 *     triangle slot) and takes the mesh as it is as the published state (it may be non-empty); the frames queued after it are
 *     recorded, on the mesh stream inside each frame's captured graph, with no host synchronisation and no allocation.  max_rows = 0
 *     turns it off and frees the buffers; enabling again starts afresh.  max_rows outside [0, 2^30], max_frames outside [1, 2^20],
 *     or a sharded handle: IMMESH_E_INVALID (immesh_mesh_shard refuses a handle with the feed on).
 *   immesh_mesh_changes(h, since_frame, ...): the frames (since_frame, newest] in order, newest = the newest frame queued; blocks
 *     until that frame has finished.  frames [n][4] = frame, v_begin, v_end, rows_end (the end of its rows in `rows`); rows [n][4];
 *     vertices [n][3] = the positions of the ids [v_begin of the first frame, v_end of the last).  counts [4] = n_frames, n_rows,
 *     n_vertices, newest_frame.  A count above its cap: IMMESH_E_CAPACITY with the counts, nothing written (caps 0: a count query).
 *     IMMESH_E_RANGE, with counts[3] = newest: since_frame is before the enable, a frame after it is no longer held (max_frames
 *     wrapped, or its rows were overwritten in the ring), or it was lost to the feed (more rows than max_rows, or more touched
 *     triangles than the per-frame list holds).  A loss never fails a push and never changes the mesh.  Resync: immesh_mesh_snapshot,
 *     then read on from counts[3] (a query with caps 0 returns it).  Not enabled, since_frame > newest, bad arguments or a sharded
 *     handle: IMMESH_E_INVALID. */
int immesh_mesh_changes_enable(immesh_mesh_t* h, int64_t max_rows, int max_frames);
int immesh_mesh_changes(immesh_mesh_t* h, int64_t since_frame, int64_t* frames /*[cap_frames][4]*/, int cap_frames, int32_t* rows /*[cap_rows][4]*/,
                        int64_t cap_rows, float* vertices /*[cap_vertices][3]*/, int64_t cap_vertices, int64_t* counts /*[4]*/);
/* The frame feed: every queued mesh frame's counters, pose, reinforced points and viewer image, recorded on the device inside the
 * frame's launch sequence (its captured graph), so that a node on the queued chain (immesh_mesh_push_frame_from_lio_async) publishes
 * per frame what the reference publishes -- the mesh_cost_time.log fields, the trajectory, the reinforced LiDAR points, a video of
 * the viewer -- without draining.  Records are numbered by the handle's frame numbers (those of immesh_mesh_changes and of
 * immesh_mesh_view_image's frame_out): frame f in header slot (f - 1) % max_frames; the frames queued after the enable are recorded.
 *   Every frame of immesh_mesh_push_frame, _dev, _from_lio, _from_lio_async, _from_lio_async_dev_n, immesh_mesh_push_depth, _depth_async and
 *     immesh_mesh_reconstruct_from_pointcloud records one frame.  A batched frame (immesh_mesh_push_frame_batched, _reconstruct_from_pointcloud_batched) records its header and pose, with
 *     no points and no image (the reinforcement and the view do not follow batched frames).
 *   header (IMMESH_MESH_FEED_HDR int64, IMMESH_MFEED_*): FRAME; KIND (IMMESH_MFEED_KIND_*); N_POINTS and STEP (append_point_step);
 *     the eight values of immesh_mesh_counts right after the frame (COUNTS + 0..7); ERR (the frame's IM_MERR flags); HAS_ROTATION (1:
 *     handed over by a localization handle); T_BEGIN_NS, T_END_NS (%globaltimer at the start of the frame's launch sequence and at its
 *     record: the device analogue of the reference's per-frame mesh time); ROW_BEGIN, ROW_END (the frame's reinforced points, numbered
 *     over the point ring) and ROWS_LOST; RF (1: the reinforcement ran for the frame); IMG_BEGIN, IMG_END (its image, numbered over the
 *     image ring: one image or none).
 *   poses (36 doubles per frame, each a row-major R then t): the frame pose (rot_end, pos_end of the handed-over state; for a
 *     world-frame push R is all zeros -- HAS_ROTATION = 0 -- and t is pose_t); the reinforcement camera as immesh_mesh_reinforced_cloud's
 *     pose_out (zeros when RF = 0); the view camera as immesh_mesh_view_image's pose_out (zeros without an image).
 *   points / pixels: the frame's reinforced points and their pixels, equal to immesh_mesh_reinforced_cloud right after the frame bit
 *     for bit and in its order.  A frame whose points exceed max_rows keeps its header and poses, sets ROWS_LOST and writes no point;
 *     a loss never fails a push and never changes the mesh.  max_rows = 0: no point is recorded (ROW_BEGIN == ROW_END, RF still set).
 *   images: the queued view's rgba (and depth with cfg.depth), equal to immesh_mesh_view_image right after the frame bit for bit; the
 *     image ring keeps the newest max_images images.  The ring is sized for the view as it is configured at the enable: every
 *     immesh_mesh_view_enable call (NULL and a new size included) turns the image recording off and frees the ring -- later frames
 *     record IMG_BEGIN == IMG_END and immesh_mesh_feed_images returns IMMESH_E_INVALID until the feed is enabled again.
 * immesh_mesh_feed_enable(h, cfg) checks its arguments, drains h, drops its captured launch sequence, frees the rings of an earlier
 *   enable and allocates everything once (an allocation failure: IMMESH_E_CAPACITY, the feed off).  NULL turns the feed off.
 *   max_frames in [1, 2^20], max_rows in [0, 2^32], max_images in [0, 2^16] (> 0 needs the queued view, immesh_mesh_view_enable),
 *   depth 0 or 1 (1 needs max_images > 0); other values or a sharded handle: IMMESH_E_INVALID.  immesh_mesh_shard refuses a handle
 *   with the feed on.  While the feed is off nothing is launched, captured or allocated for it.
 * immesh_mesh_feed(h, since_frame, wait, ...) returns the frames (since_frame, newest finished] oldest first, their poses (or NULL)
 *   and their points and pixels concatenated (or NULL; pixels are written with points); immesh_mesh_feed_images the same frames'
 *   headers and the images they hold, concatenated oldest first (rgba or depth may be NULL).  wait = 0 never blocks on queued work
 *   ("finished": a pinned host word the last kernel of each record writes; the copies run on a stream of the feed's own); wait = 1
 *   first waits for the newest queued frame's record only.  counts [4] = frames, rows (images), newest finished, newest queued.
 *   cap_frames (cap_images) = 0: a count query.  More frames than the cap, or more points than cap_rows: IMMESH_E_CAPACITY with the
 *   counts, nothing written.  IMMESH_E_RANGE with counts[2] set (read on from there): the range reaches back before the enable, or a
 *   slot of it (header, points or image) was overwritten before or during the copy.  Bad arguments, the feed off, since_frame newer
 *   than the newest queued frame, images requested while image recording is off, depth requested without cfg.depth, or a sharded
 *   handle: IMMESH_E_INVALID.  A record kernel that computes a slot outside its ring (an internal error) writes nothing and the push
 *   that harvests the frame returns IMMESH_E_CUDA ("internal error"). */
typedef struct {
    int64_t max_frames;   /* header + pose ring, in frames: [1, 2^20] */
    int64_t max_rows;     /* reinforced-point ring, rows: [0, 2^32]; 0 = no points recorded */
    int64_t max_images;   /* view image ring, in images: [0, 2^16]; > 0 needs the queued view enabled */
    int depth;            /* 1: the image ring also keeps the view's depth image */
    int pad;
} immesh_mesh_feed_config;
#define IMMESH_MESH_FEED_HDR 22
#define IMMESH_MESH_FEED_POSE 36
#define IMMESH_MFEED_FRAME 0
#define IMMESH_MFEED_KIND 1
#define IMMESH_MFEED_N_POINTS 2
#define IMMESH_MFEED_STEP 3
#define IMMESH_MFEED_COUNTS 4   /* 8 fields: immesh_mesh_counts' out[0..7] */
#define IMMESH_MFEED_ERR 12
#define IMMESH_MFEED_HAS_ROTATION 13
#define IMMESH_MFEED_T_BEGIN_NS 14
#define IMMESH_MFEED_T_END_NS 15
#define IMMESH_MFEED_ROW_BEGIN 16
#define IMMESH_MFEED_ROW_END 17
#define IMMESH_MFEED_ROWS_LOST 18
#define IMMESH_MFEED_RF 19
#define IMMESH_MFEED_IMG_BEGIN 20
#define IMMESH_MFEED_IMG_END 21
/* IMMESH_MFEED_KIND: the entry point that queued the frame */
#define IMMESH_MFEED_KIND_PUSH 0
#define IMMESH_MFEED_KIND_PUSH_DEV 1
#define IMMESH_MFEED_KIND_FROM_LIO 2
#define IMMESH_MFEED_KIND_FROM_LIO_ASYNC 3
#define IMMESH_MFEED_KIND_RECONSTRUCT 4
#define IMMESH_MFEED_KIND_BATCHED 5
#define IMMESH_MFEED_KIND_RECONSTRUCT_BATCHED 6
#define IMMESH_MFEED_KIND_DEPTH 7   /* immesh_mesh_push_depth and _async */
#define IMMESH_MFEED_KIND_FROM_LIO_ASYNC_DEV_N 8   /* immesh_mesh_push_frame_from_lio_async_dev_n */
int immesh_mesh_feed_enable(immesh_mesh_t* h, const immesh_mesh_feed_config* cfg /* NULL: off */);
int immesh_mesh_feed(immesh_mesh_t* h, int64_t since_frame, int wait, int64_t* frames /*[cap_frames][22]*/, double* poses /*[cap_frames][36] or NULL*/,
                     int cap_frames, float* points /*[cap_rows][3] or NULL*/, int32_t* pixels /*[cap_rows] or NULL*/, int64_t cap_rows, int64_t* counts /*[4]*/);
int immesh_mesh_feed_images(immesh_mesh_t* h, int64_t since_frame, int wait, int64_t* frames /*[cap_images][22]*/, int cap_images,
                            uint8_t* rgba /*[cap_images][h][w][4] or NULL*/, float* depth /*[cap_images][h][w] or NULL*/, int64_t* counts /*[4]*/);
/* Evaluation of the mesh against a ground-truth cloud with the metrics of the ImMesh paper's Experiment-3 (section VIII-C, Tables V
 * and VI, Fig. 8 and 9): fairness (mean Max-Min interior angle, mean circumradius-to-shortest-edge ratio) and correctness (accuracy,
 * completeness, precision, recall, F-score between points sampled on the mesh and the down-sampled ground truth).
 *   Positions: float32, the raw vertex positions (positions = 0, as immesh_mesh_snapshot) or (float) of the stored smoothed positions
 *     (positions = 1, what save_to_ply_file writes with smooth_factor != 0).  positions = 1 with a vertex of a live triangle whose
 *     m_smoothed flag is clear: IMMESH_E_INVALID ("smooth first"; immesh_mesh_smooth_all sets every flag).  The call smooths nothing.
 *   Fairness, per live triangle in float64: the interior angles atan2(|u x v|, u . v) in degrees; C2SE = |a||b||c| / (2 |AB x AC|) /
 *     shortest edge.  A triangle with |AB x AC| == 0 is degenerate: counted, left out of both means, and given no samples.
 *   Mesh samples: with A < B < C the vertex ids and n = max(1, ceil(longest edge / sample_spacing)), the centroids of the n^2
 *     sub-triangles of the n-subdivision: "up" at barycentrics ((3i+1)/(3n), (3j+1)/(3n)), i in [0, n), j in [0, n-i), and "down" at
 *     ((3i+2)/(3n), (3j+2)/(3n)), j in [0, n-i-1); sample = (float)(A + (u (B-A) + v (C-A))) in float64 without FMA.  Every sample
 *     lies inside exactly one facet: none is repeated along a shared edge.  A triangle that needs n > 2^15: IMMESH_E_RANGE.
 *   Ground truth: gt_leaf > 0: leaf key floor((double)p / gt_leaf) (int64, per axis); every occupied leaf gives one point,
 *     (float)(sum of (double)p / count) with the sum taken in input order.  There is no index-overflow pass-through (unlike
 *     pcl::VoxelGrid): a 1 cm leaf over a city down-samples.  gt_leaf = 0: every point as given.  A non-finite point: IMMESH_E_INVALID.
 *     At most 2^31 - 1 points per call (IMMESH_E_RANGE).
 *   Distances: d = sqrt((dx dx + dy dy) + dz dz) in float64 from the float32 coordinates, the exact minimum over the other set's points
 *     within max_dist (d <= max_dist).  A query with none takes d = max_dist and is "far".  d is quantised to q = rint(d 2^20) and
 *     summed in int64 (q <= 2^30, at most 2^33 samples, else IMMESH_E_RANGE): the sums do not depend on order, batching or tiling and
 *     compare exactly.  "Within" is d < threshold (strict).
 *   counts [12]: live triangles, degenerate triangles, samples, ground-truth points after down-sampling, samples within, ground-truth
 *     points within, far samples, far ground-truth points, incorrect facets, sum q over the samples, sum q over the ground truth,
 *     subdivisions n of the largest triangle.
 *   metrics [8] (float64): mean Max-Min angle (degrees), mean C2SE, accuracy (m) = sum q / 2^20 / samples, completeness (m) = sum q /
 *     2^20 / ground-truth points, precision = samples within / samples, recall = ground-truth points within / ground-truth points,
 *     F-score = 2 P R / (P + R) (0 when P + R = 0), 0 (spare).  A mean over an empty set is NaN (and so is an F-score with one).
 *     Accuracy and completeness are lower bounds when the far counts are non-zero: a far query counts max_dist, not its distance.
 *   facet_rows [cap_rows][5] (or NULL: none): one row a b c n_samples n_far per live triangle in ascending (a, b, c) order (the change
 *     feed's order), n_far = its samples not within threshold.  A facet is incorrect (paper Fig. 8) when n_samples > 0 and
 *     n_far >= incorrect_ratio * n_samples.  *n_rows (or NULL) = live triangles.  facet_rows given and cap_rows below the live count:
 *     IMMESH_E_CAPACITY before any work, nothing else written (cap_rows = 0: the count query).
 *   Contract: blocks; drains the frames queued on h first, those of immesh_mesh_push_frame_from_lio_async included.  Changes nothing
 *     on the handle (vertices, flags, smoothed positions, counters, captured graphs).  The ground truth is read in place (on_device = 1,
 *     a device pointer) or copied to the device once.  Every other device buffer is allocated by the call and freed before it returns,
 *     at most max_batch_bytes in all (0: 2 GiB): one block for the table (about 110 bytes per live triangle, 130 with the rows), then one
 *     block the size of the largest tile's scratch, reused by every tile.  A tile is a box of the bisected bounding box; its scratch holds
 *     the samples and ground-truth points of the box grown by max_dist, with their hashed grids.  Tiles are halved until each fits
 *     what the table leaves of the budget.  A budget too small for the table, or for a tile that cannot be halved further (side
 *     max(max_dist / 4, 2 grid cells)): IMMESH_E_CAPACITY, naming it.  A configuration whose smallest tile would span more than
 *     2^21 - 4 grid cells or ground-truth leaves per axis (gt_leaf far below max_dist, or coordinates beyond about 10^6 m):
 *     IMMESH_E_RANGE before any tile is processed.
 *   immesh_mesh_evaluate_stats(out[4]): what the calling thread's last immesh_mesh_evaluate that got past its argument checks did:
 *     tiles processed, boxes counted by the tile planner, device scratch bytes (table + tile block, the ground-truth copy excluded),
 *     table bytes.
 *   IMMESH_E_INVALID: NULL h, cfg, counts or metrics; sample_spacing <= 0; gt_leaf < 0; not 0 < threshold <= max_dist <= 1024;
 *     incorrect_ratio outside (0, 1]; positions not 0 or 1; max_batch_bytes < 0; n_gt < 0 or gt_xyz NULL with n_gt > 0; a non-finite
 *     configuration value; a sharded handle. */
typedef struct {
    double sample_spacing;    /* mesh sampling step (paper: 0.01 m), > 0 */
    double gt_leaf;           /* ground-truth down-sampling leaf (paper: 0.01 m); 0 = every point as given */
    double threshold;         /* precision / recall / correct-sample distance (paper: 0.05 m), > 0 */
    double max_dist;          /* nearest-neighbour search radius, threshold <= max_dist <= 1024 */
    double incorrect_ratio;   /* facet incorrect when n_far >= ratio * n_samples (paper Fig. 8: 0.8), in (0, 1] */
    int positions;            /* 0: raw vertex positions (immesh_mesh_snapshot); 1: smoothed (what save_to_ply_file writes, smooth_factor != 0) */
    int pad;
    int64_t max_batch_bytes;  /* scratch budget of the call beyond the ground-truth copy; 0 = a default (2 GiB) */
} immesh_eval_config;
int immesh_mesh_evaluate(immesh_mesh_t* h, const float* gt_xyz /*[n_gt][3]*/, int64_t n_gt, int on_device, const immesh_eval_config* cfg,
                         int64_t* counts /*[12]*/, double* metrics /*[8]*/, int32_t* facet_rows /*[cap_rows][5] or NULL*/, int64_t cap_rows,
                         int64_t* n_rows /*or NULL*/);
int immesh_mesh_evaluate_stats(int64_t* out /*[4]*/);
/* The textured mesh of the paper (ImMesh, Fig. 1(b, c), Fig. 11, Application-2 in section VIII-E: "each facet of the reconstructed mesh
 * textured by the RGB image captured by the nearest camera frame with the estimated camera pose"): for every live triangle, the
 * camera that textures it and the pixel coordinates of its corners in that camera's image.  No pixel is resampled: the export
 * (immesh_write_obj_textured) points at the caller's image files.
 *   immesh_mesh_texture_select: blocking, on the mesh stream behind the frames already queued (those of
 *     immesh_mesh_push_frame_from_lio_async included).  It reads the mesh and writes nothing on the handle (no smoothed position,
 *     m_smoothed flag, counter or change-feed row), as immesh_mesh_render_view.
 *   Rows: one per live triangle in immesh_mesh_snapshot's order (row i is snapshot triangle i), as immesh_mesh_evaluate's facet rows.
 *     facet_cam [cap]: the chosen camera, -1 for none; facet_uv [cap][6]: u0 v0 u1 v1 u2 v2 of the corners q0 q1 q2 (below) in the
 *     chosen camera's pixels, left unwritten where facet_cam = -1; facet_px [cap][2]: won and covered (below) of the chosen camera,
 *     0 0 where facet_cam = -1; vertices [n_vertices][3]: the positions the rule used (cfg.positions), n_vertices as immesh_mesh_counts
 *     reports it after immesh_mesh_wait (the call includes the queued frames' vertices).  Each may be NULL.
 *     *n_facets = the live triangle count; above cap: IMMESH_E_CAPACITY and nothing written (cap = 0: a count query).
 *     counts [4] (or NULL): facets textured, facets untextured, cameras that texture at least one facet, pixels rasterised (the sum
 *     of width * height over the cameras).
 *   Selection rule (defined here), float64 in the order written, without fused multiply-adds.  A facet's corners q0 q1 q2 are its
 *     stored triple's positions p0 p1 p2 at cfg.positions (immesh_view_style.positions: 0 raw, 1 the smoothed position as float where
 *     m_smoothed is set) in immesh_write_ply's face order: m_index_flip != 0 p0 p1 p2, else p0 p2 p1.
 *     1. Camera: the OpenCV camera (x right, y down, z forward; world = cam_R p + cam_t) is the rasteriser's camera of
 *        immesh_mesh_render_depth with columns 1 and 2 of cam_R negated, an exact conversion.
 *     2. Visible pixels: immesh_mesh_render_view's visibility rule unchanged at that camera and positions, with cfg's z range: samples
 *        at integer pixels, the edge-function cover (zero included), 1/z affine, a triangle with a corner outside (z_near, z_far)
 *        skipped; at each pixel the smaller depth bits win, then the lower (a, b, c) triple.  covered_k(f): the pixels where f has a
 *        sample; won_k(f): the pixels f wins.
 *     3. Seen by camera k: every corner projects into [0, w - 1] x [0, h - 1]; won >= 1; 1000 won >= min_visible_permille covered;
 *        and with g = ((q0 + q1) + q2) / 3, e = cam_t - g, n = (q1 - q0) x (q2 - q0), s = (n0 e0 + n1 e1) + n2 e2: s > 0 (the camera on
 *        the oriented front side; two_sided: s != 0), and s s >= (min_cos min_cos) (|n|^2 |e|^2), squared norms summed (x^2 + y^2) + z^2.
 *     4. Nearest: of the cameras that see f, the smallest |e|^2; on a tie the lower camera index.  None: facet_cam = -1.
 *     5. UVs: the chosen camera's pixel coordinates (u, v) of q0, q1, q2, as (float) of the float64 projection.
 *     The cameras run one after another in index order and each facet is updated by one thread with a strict <, so the result does
 *     not depend on atomics or scheduling.
 *   IMMESH_E_INVALID: NULL h, cams, cfg or n_facets; n_cams < 1; a camera with a size outside [1, 2^26] pixels, non-finite
 *     intrinsics or pose, or fx or fy = 0; not 0 < z_near < z_far < inf; min_cos outside [0, 1]; min_visible_permille outside
 *     [0, 1000]; two_sided or positions not 0 / 1; cap < 0; a sharded handle.
 *   Lens distortion is not modelled: pass rectified images.  Intrinsics scaled to a smaller image select at that resolution; the
 *   export's normalised coordinates then texture with the full-size images.
 * immesh_write_obj_textured: host-side only, a Wavefront OBJ + MTL pair of the rows above (vertices, triangles and flips as
 *   immesh_mesh_snapshot returns them, or the vertices texture_select wrote).  The OBJ: "mtllib <mtl_path's file name>", one "v x y z"
 *   per vertex (%.9g), three "vt s t" per textured facet with s = (u + 0.5) / W, t = 1 - (v + 0.5) / H of its camera's size (pixel
 *   centres at integers, so the coordinates do not depend on the resolution selected at), then the faces grouped by "usemtl tex_<k>"
 *   in ascending k with the rows in order inside a group, each "f a/ta b/tb c/tc" (1-based) with the corners in the face order q0 q1
 *   q2; the untextured facets last under "usemtl untextured", as "f a b c".  The MTL: "newmtl tex_<k>" with "map_Kd <image_files[k]>"
 *   for every camera that textures a facet, and "newmtl untextured".  A triangle index outside [0, nv): IMMESH_E_RANGE; facet_cam
 *   outside [-1, n_cams), a camera size below 1, a NULL image file of a used camera, or a file that cannot be written:
 *   IMMESH_E_INVALID. */
typedef struct {
    int width, height;            /* image size in pixels, [1, 2^26] pixels */
    double fx, fy, cx, cy;        /* pinhole intrinsics, finite, fx and fy != 0 */
    double cam_R[9], cam_t[3];    /* camera to world, row-major, OpenCV axes (x right, y down, z forward), as immesh_depth_frame */
} immesh_texture_camera;
typedef struct {
    double z_near, z_far;         /* 0 < z_near < z_far < inf */
    double min_cos;               /* [0, 1]: the least |cos| between the facet normal and the view ray */
    int min_visible_permille;     /* [0, 1000]: the least share of the facet's covered pixels it must win */
    int two_sided;                /* 0: only cameras on the oriented front side; 1: either side */
    int positions;                /* as immesh_view_style.positions: 0 raw, 1 smoothed where m_smoothed is set */
    int pad;
} immesh_texture_config;
int immesh_mesh_texture_select(immesh_mesh_t* h, const immesh_texture_camera* cams, int n_cams, const immesh_texture_config* cfg,
                               int32_t* facet_cam /*[cap] or NULL*/, float* facet_uv /*[cap][6] or NULL*/,
                               int32_t* facet_px /*[cap][2] or NULL: won, covered in the chosen camera*/,
                               float* vertices /*[n_vertices][3] or NULL: the positions used*/,
                               int64_t cap, int64_t* n_facets, int64_t* counts /*[4] or NULL: textured, untextured, cameras used, pixels rasterised*/);
/* Texturing queued behind every frame: each triangle record keeps the nearest frame whose camera sees it, updated on the device at the
 * end of every queued frame, so a textured mesh can be read at any moment and the images no frame textures any more can be deleted.
 *   immesh_mesh_texture_enable(h, rig, cfg): rig = the colour camera (immesh_texture_camera: width, height, fx, fy, cx, cy; cam_R, cam_t
 *     its pose in the frame's sensor frame, OpenCV axes: the localization state's body frame for a frame handed over by a localization
 *     handle, the depth camera for a depth frame); cfg = immesh_mesh_texture_select's config with positions = 0 (the raw positions).
 *     As the other queued stages it drains the handle, drops the captured launch sequence and allocates everything once; every triangle
 *     record starts unobserved (enabling again starts afresh).  rig = NULL turns it off and frees the state; off, nothing is launched,
 *     captured or allocated.  The state is 48 + 8 bytes per triangle slot of the pool's capacity (1.75 GiB at 32 Mi slots), allocated
 *     for the current capacity and grown with the triangle pool.
 *   immesh_mesh_texture_pose(h, cam_R, cam_t): from the next queued frame on, (cam_R, cam_t) (finite, camera to world, OpenCV axes) is the
 *     camera of every frame, with the rig's size and intrinsics; NULL, NULL returns to the rig (the mode after enable).
 *   Camera of frame f (f the handle's frame number), float64 in the order written without fused multiply-adds: with the sensor pose
 *     (R_f, t_f), R = R_f R_rig (each entry (R_f[r][0] R_rig[0][c] + R_f[r][1] R_rig[1][c]) + R_f[r][2] R_rig[2][c]) and
 *     t = ((R_f[r][0] t_rig0 + R_f[r][1] t_rig1) + R_f[r][2] t_rig2) + t_f[r].  (R_f, t_f) is the converged (rot_end, pos_end) for
 *     immesh_mesh_push_frame_from_lio, _async and _async_dev_n, and the depth frame's cam_R, cam_t for immesh_mesh_push_depth and
 *     _async.  World-frame pushes (immesh_mesh_push_frame, _dev, immesh_mesh_reconstruct_from_pointcloud) have no sensor rotation:
 *     no camera, the frame is not observed, unless a caller camera is set.  Batched frames are never observed.
 *   Update, at the end of frame f (after its push) when it has a camera C_f: every triangle record live then gets won and covered at
 *     C_f by immesh_mesh_texture_select's rule (steps 1-3, raw positions, cfg's z range, the record's current flip for the face order
 *     and the front-side test); when seen with |e|^2 < the record's stored |e|^2 (strict: a tie keeps the earlier frame), the record
 *     stores (f, |e|^2, won, covered, uv) with uv the corners' pixel coordinates in stored (ascending vertex id) order.  Records that are
 *     not live keep their state: a record that comes back is the same three vertices, which never move.
 *   immesh_mesh_texture_rows: blocking, on the mesh stream behind the queued frames; writes nothing on the handle.  One row per live
 *     triangle in immesh_mesh_snapshot's order, in texture_select's layout: facet_cam = the chosen frame number or -1; facet_uv the
 *     stored uv in the current face order, unwritten for -1 rows; facet_px won, covered at that frame (0 0 for -1).  counts [4]:
 *     textured rows, untextured rows, distinct frames of the live rows, pixels rasterised since the enable (w h per frame with a
 *     camera).  frames [cap_frames]: the ascending distinct frames of every record, live or not (the images still needed), *n_frames
 *     their number.  *n_facets above cap or (frames given) *n_frames above cap_frames: IMMESH_E_CAPACITY with the counts, nothing else
 *     written (0: a count query).  The rows go to immesh_mesh_texture_bake and immesh_write_obj_textured with the cameras indexed by
 *     frame number.
 *   IMMESH_E_INVALID: NULL h; a rig or cfg texture_select refuses, or positions != 0; cam_R / cam_t or frames / n_frames given one
 *     without the other; NULL n_facets; cap or cap_frames < 0; texture_pose or texture_rows while off; a sharded handle
 *     (immesh_mesh_shard refuses a handle with the texturing on). */
int immesh_mesh_texture_enable(immesh_mesh_t* h, const immesh_texture_camera* rig /* NULL: off */, const immesh_texture_config* cfg);
int immesh_mesh_texture_pose(immesh_mesh_t* h, const double* cam_R /*[9] or NULL*/, const double* cam_t /*[3] or NULL*/);
int immesh_mesh_texture_rows(immesh_mesh_t* h, int32_t* facet_cam /*[cap] or NULL*/, float* facet_uv /*[cap][6] or NULL*/,
                             int32_t* facet_px /*[cap][2] or NULL*/, int64_t cap, int64_t* n_facets, int64_t* counts /*[4] or NULL*/,
                             int32_t* frames /*[cap_frames] or NULL*/, int64_t cap_frames, int64_t* n_frames /*or NULL*/);
int immesh_write_obj_textured(const char* obj_path, const char* mtl_path, const float* vertices /*[nv][3]*/, int nv,
                              const int32_t* triangles /*[nt][3]*/, const int32_t* flips /*[nt] or NULL*/, const int32_t* facet_cam /*[nt]*/,
                              const float* facet_uv /*[nt][6]*/, int nt, const int32_t* cam_wh /*[n_cams][2]*/, const char* const* image_files /*[n_cams]*/,
                              int n_cams);
/* The texture atlas of a selection: every textured facet's pixels resampled out of its chosen image into a few square pages, so the
 * textured mesh ships as one OBJ, one MTL and n_pages images instead of pointing at every source image.
 *   immesh_mesh_texture_bake: blocking, on the mesh stream behind the frames already queued.  It reads nothing from the mesh: h gives
 *     the device and the stream, and nothing on the handle is written.  Input: immesh_mesh_texture_select's rows as they are
 *     (facet_cam [n_facets], facet_uv [n_facets][6] in the selection camera's pixels), cams (only width and height are read) and one
 *     image per camera (data NULL for a camera no facet uses).  on_device 1: every data pointer is device memory of h's device; 0:
 *     host memory, uploaded in camera index order in batches of whole images, each batch at most cfg.max_image_bytes bytes (packed
 *     3 width height), into two alternating device arenas of that size, so the next batch's copy overlaps this batch's bake.
 *   Outputs: facet_page [n_facets]: the page of the facet's cell, -1 where facet_cam = -1; atlas_uv [n_facets][6]: u0 v0 u1 v1 u2 v2 of
 *     the corners in page texels (centres at integers), left as the caller had them where facet_cam = -1; pages [n_pages][P][P][3]
 *     (P = cfg.page_size, rows top to bottom, the images' channel order); *n_pages; counts [4]: textured rows, untextured rows, cells,
 *     texels written.  pages = NULL: a count query, which lays out the atlas only (facet_page, atlas_uv, *n_pages, counts).
 *     n_pages > cap_pages with pages != NULL: IMMESH_E_CAPACITY with *n_pages set and nothing written.  Each other output may be NULL.
 *   Export: immesh_write_obj_textured with facet_page as facet_cam, atlas_uv as facet_uv, (P, P) as every cam_wh and the pages'
 *     image files (immesh_write_png) as image_files; untextured facets land in its "untextured" material.
 *   Atlas rule (defined here), float64 in the order written, without fused multiply-adds:
 *     1. Scale: a textured row's corners in its image (W x H, the selection camera Ws x Hs): u' = ((u + 0.5) W) / Ws - 0.5,
 *        v' = ((v + 0.5) H) / Hs - 0.5.
 *     2. Cell: L = the longest of the three edges sqrt(du du + dv dv) of (u', v'); the cell side S is the smallest power of two >= 8
 *        and >= ceil(L) + 4, or cfg.max_cell if that is smaller.  class = log2 S.
 *     3. Order: the textured rows sorted stably by (class descending, camera ascending); rows keep their input order inside a key.
 *        Consecutive rows of a class share a cell: the class's q-th row (from 0) takes cell q / 2, slot q % 2.
 *     4. Slots: texel (i, j) of a cell (i the column, j the row, 0 <= i, j < S) belongs to slot 0 when i + j <= S - 2, else to slot 1.
 *        The triangle of slot 0 is (0, 0), (S - 4, 0), (0, S - 4); that of slot 1 is (S - 2, S - 2), (2, S - 2), (S - 2, 2); row
 *        corner k maps to triangle corner k.  Every texel a bilinear lookup anywhere inside a slot's triangle touches belongs to that
 *        slot and lies in the cell, so seams do not bleed at the base level (mip-maps may bleed across cells).
 *     5. Placement: cells in sorted order, class by class; a cell's offset is the exclusive sum of (S / 8)^2 over the cells before it,
 *        in 8 x 8-texel units.  With U = (P / 8)^2 units per page, the cell is on page offset / U at texel (8 x, 8 y), where x (the even
 *        bits) and y (the odd bits) are the Morton decode of offset % U.  Sides only shrink, so cells are aligned and none straddles a
 *        page.  n_pages = ceil(total units / U).  atlas_uv of a row: its cell's origin plus its slot's triangle corners.
 *     6. Texel (i, j) of a filled slot, T = S - 4: w1 = i / T, w2 = j / T (slot 1: w1 = (S - 2 - i) / T, w2 = (S - 2 - j) / T);
 *        a = max(w1, 0), b = max(w2, 0); if a + b > 1: s = a + b, a = a / s, b = b / s; w0 = (1 - a) - b.  The source point is
 *        x = (w0 u'0 + a u'1) + b u'2 and the same for y, clamped to [0, W - 1] x [0, H - 1].  With x0 = floor(x), x1 = min(x0 + 1,
 *        W - 1), fx = x - x0 (y likewise), each channel is (1 - fy) ((1 - fx) I(x0, y0) + fx I(x1, y0)) + fy ((1 - fx) I(x0, y1) +
 *        fx I(x1, y1)), written as floor(value + 0.5).  Texels no filled slot owns are 0.
 *   IMMESH_E_INVALID: NULL h, cams, images, cfg or n_pages; n_cams outside [1, 2^27); n_facets outside [0, 2^31) (or > 0 with NULL
 *     facet_cam or facet_uv); on_device not 0 / 1; page_size not a power of two in [256, 8192]; max_cell not a power of two in [8, page_size];
 *     max_image_bytes < 0; a facet_cam outside [-1, n_cams); a textured row with a non-finite uv; a used camera with a NULL image,
 *     an image or camera size below 1, a pitch below 3 width, or (host images) an image larger than max_image_bytes; cap_pages < 0.
 * immesh_write_png: host only.  An 8-bit RGB PNG of rgb [height][width][3] (rows top to bottom), uncompressed: stored deflate blocks,
 *   CRC-32 and Adler-32 computed in place, so no compression library is needed.  IMMESH_E_INVALID: NULL path or rgb, a size below 1,
 *   or a file that cannot be written. */
typedef struct {
    const uint8_t* data;   /* 8-bit, 3 interleaved channels (any order: the pages keep it); NULL for a camera no facet uses */
    int width, height;     /* may differ from the selection camera's: texture coordinates are rescaled */
    int64_t pitch;         /* bytes per row, >= 3 * width */
} immesh_texture_image;
typedef struct {
    int page_size;             /* texels per page side: a power of two in [256, 8192] */
    int max_cell;              /* the largest cell: a power of two in [8, page_size] */
    int64_t max_image_bytes;   /* host images: device bytes of each of the two upload arenas (0: 512 MiB); must hold the largest used image */
} immesh_texture_atlas_config;
int immesh_mesh_texture_bake(immesh_mesh_t* h, const immesh_texture_camera* cams /* the selection's cameras: width, height */, int n_cams,
                             const immesh_texture_image* images /*[n_cams]*/, int on_device,
                             const int32_t* facet_cam /*[n]*/, const float* facet_uv /*[n][6]*/, int64_t n_facets,
                             const immesh_texture_atlas_config* cfg,
                             uint8_t* pages /*[cap_pages][page][page][3] or NULL*/, int cap_pages,
                             int32_t* facet_page /*[n] or NULL*/, float* atlas_uv /*[n][6] or NULL*/,
                             int* n_pages, int64_t* counts /*[4] or NULL: textured, untextured, cells, texels written*/);
int immesh_write_png(const char* path, const uint8_t* rgb /*[h][w][3]*/, int width, int height);
/* The textured mesh rendered at any camera, and scored against a photo taken there: a preview without a display or an external viewer,
 * and the photometric measure of texture quality (render at a camera whose photo was held out of the texturing, compare with it).
 *   immesh_mesh_render_textured: blocking, on the mesh stream behind the frames already queued; it reads the mesh and writes nothing on
 *     the handle.  Input: rows of any of the three producers, one per live triangle in immesh_mesh_snapshot's order -- texture_select's
 *     (facet_cam, facet_uv) with its cameras and images; texture_rows' with cameras and images indexed by frame number; or the bake's
 *     (facet_page, atlas_uv) with (P, P) cameras and the pages as images.  cams: only width and height are read (the size the uv were
 *     made at); images [n_cams] as immesh_mesh_texture_bake's (on_device 1: device memory of h's device, 0: host memory uploaded in
 *     camera order through two alternating arenas of cfg.max_image_bytes), but only the cameras the view samples are read: an entry
 *     may be NULL for any other.  truth (or NULL): a photo at the view's size, in the same memory as the images.
 *   Outputs, each may be NULL: rgb [h][w][3]; depth [h][w]; facet [h][w] the winning triangle's snapshot row, -1 where no triangle has
 *     a sample; needed [n_cams] 1 where some pixel samples camera k, else 0; counts [8]: pixels won by a textured row, pixels won by an
 *     untextured row (facet_cam = -1), pixels without a sample, cameras sampled, then with truth the sums over the textured pixels of
 *     (rgb - truth)^2 for channels 0, 1 and 2 and of |rgb - truth| over all three channels (0 without truth).  Every count is an integer
 *     sum, so the result does not depend on atomics or scheduling.
 *   images = NULL: a query.  It resolves visibility and writes depth, facet, needed and counts [0, 4) (rgb and truth must be NULL): a
 *     caller whose images live on disk by frame number loads only the needed ones.
 *   Pixel rule (defined here), float64 in the order written, without fused multiply-adds:
 *     1. Camera: view is an OpenCV camera, converted to the rasteriser's exactly as texture_select's step 1.
 *     2. Visibility: immesh_mesh_render_view's rule unchanged at cfg's z range and positions; the nearest depth bits win, then the
 *        lower (a, b, c) triple.  depth is immesh_mesh_render_view's depth image at that camera bit for bit (-1 at or beyond 0.99 z_far
 *        or without a sample).
 *     3. Weights: the winner's set-up with its corners p0 p1 p2 in stored (ascending id) order, w_i = e_i (1 / z_i) from the sample's
 *        edge functions, as render_view's shading.
 *     4. Face order: the row's corners are q0 q1 q2 of immesh_write_ply's face order, so o0 = w0, o1 = flip ? w1 : w2,
 *        o2 = flip ? w2 : w1 with flip the triangle's current m_index_flip.
 *     5. Source point: the row's uv scaled to image k = facet_cam[row] (W x H, cams[k] Ws x Hs) by the bake's rule 1:
 *        u'_j = ((u_j + 0.5) W) / Ws - 0.5, v'_j likewise; x = ((o0 u'0 + o1 u'1) + o2 u'2) / ((o0 + o1) + o2), y likewise.  This is
 *        the perspective-correct interpolation an OBJ viewer applies to immesh_write_obj_textured's output, pixel centres at integers.
 *     6. Sample: the bake's rule 6 at (x, y): clamped to [0, W - 1] x [0, H - 1], bilinear, each channel floor(value + 0.5).
 *     7. Colour: a pixel won by a textured row gets its sample; won by an untextured row, cfg.untextured; without a sample,
 *        cfg.background.  As in render_view, a pixel with a sample is coloured even where its depth is -1 beyond 0.99 z_far.
 *   IMMESH_E_INVALID, nothing written: NULL h, view, cfg or cams; n_cams < 1; a view texture_select refuses as a camera; not 0 <
 *     z_near < z_far < inf, positions not 0 / 1 or max_image_bytes < 0; on_device not 0 / 1; n_facets other than the live triangle
 *     count (rows of another mesh state; their match beyond the count is the caller's contract, as for the bake and the export) or
 *     > 0 with NULL rows; a facet_cam outside [-1, n_cams) or a textured row with a non-finite uv; a given image of a used camera that
 *     the bake refuses (size or camera size below 1, pitch below 3 width, a host image larger than max_image_bytes); a NULL image for a
 *     camera the view samples; a truth image not of the view's size or with a pitch below 3 width; rgb or truth with images = NULL; a
 *     sharded handle. */
typedef struct {
    double z_near, z_far;        /* the view's z range: 0 < z_near < z_far < inf */
    int positions;               /* 0 raw, 1 the smoothed position where m_smoothed is set: pass the rows' own setting */
    uint8_t untextured[3];       /* a pixel won by an untextured facet, e.g. (128, 128, 128): the MTL's Kd 0.5 */
    uint8_t background[3];       /* a pixel without a sample, e.g. (0, 0, 0): the viewer's clear colour */
    int64_t max_image_bytes;     /* host images: bytes of each of the two upload arenas (0: 512 MiB); must hold the largest needed image */
} immesh_texture_view_config;
int immesh_mesh_render_textured(immesh_mesh_t* h, const immesh_texture_camera* view, const immesh_texture_view_config* cfg,
                                const immesh_texture_camera* cams /* width, height */, int n_cams, const immesh_texture_image* images /*[n_cams] or NULL*/,
                                int on_device, const int32_t* facet_cam /*[n_facets]*/, const float* facet_uv /*[n_facets][6]*/, int64_t n_facets,
                                const immesh_texture_image* truth /* or NULL */, uint8_t* rgb /*[h][w][3] or NULL*/, float* depth /*[h][w] or NULL*/,
                                int32_t* facet /*[h][w] or NULL*/, uint8_t* needed /*[n_cams] or NULL*/, int64_t* counts /*[8] or NULL*/);
/* The phases of this thread's last successful immesh_mesh_render_textured, in milliseconds from CUDA events on the mesh stream:
 * ms [3] = pass A (snapshot order, binning, tiles), pass B (with host images the uploads it waits for included), score (with a host
 * truth image its upload included). */
int immesh_mesh_render_textured_stats(double* ms /*[3]*/);
/* Colour equalisation between cameras: each facet takes its colour from one camera, and each camera has its own exposure and white
 * balance, so the textured mesh shows brightness steps wherever neighbouring facets chose different cameras.  Gain compensation in the
 * style of Brown & Lowe (panorama stitching, OpenCV's GainCompensator) solves one gain per camera and channel so that cameras agree
 * where they see the same surface; the mesh gives that overlap exactly: a facet that camera k sees and camera c textures.
 *   immesh_mesh_texture_gains: blocking, on the mesh stream behind the frames already queued; it reads the mesh and writes nothing on
 *     the handle.  Input: the rows of texture_select or texture_rows (facet_cam, facet_uv, n_facets = the live triangle count), before
 *     any bake; cams [n_cams] full cameras indexed as the rows index them (by frame number for texture_rows); images [n_cams] as
 *     immesh_mesh_texture_bake's (on_device 1: device memory of h's device; 0: host memory uploaded in camera order through two
 *     alternating arenas of cfg.max_image_bytes); a NULL image: the camera takes no part in the solve.  cfg.sel is the select rule
 *     that decides whether an observer sees a facet: pass the rows' own positions.
 *   Outputs: gains [n_cams][3] (float64, channel order of the images); pair_cam [max_pairs][2] (k, c) and pair_sums [max_pairs][7]
 *     (n, S_k[3], S_c[3]) or NULL; *n_pairs (or NULL); counts [8] (or NULL): pairs, sample pairs used, sample pairs clipped, observer
 *     cameras rasterised, cameras left at gain 1, CG iterations (the most over the three channels), pixels rasterised (w h summed over
 *     the observers), 0.  *n_pairs > cfg.max_pairs: IMMESH_E_CAPACITY with *n_pairs and counts set, no gain or pair written.
 *   Rule (defined here), float64 in the order written, without fused multiply-adds:
 *     1. Sample points: the 10 barycentric points (b0, b1, b2) = (i / 6, j / 6, l / 6) with i, j, l >= 1, i + j + l = 6, in the order
 *        i = 1..4, then j = 1..5 - i (l = 6 - i - j), applied to the corners in the row's face order q0 q1 q2.
 *     2. Chosen side: row f with c = facet_cam[f] >= 0: its uv scaled to image c by the bake's rule 1 (W x H the image, Ws x Hs =
 *        cams[c]'s size), the point x = (b0 u'0 + b1 u'1) + b2 u'2, y likewise, read at the nearest pixel (floor(x + 0.5), floor(y +
 *        0.5)) clamped to [0, W - 1] x [0, H - 1]: 10 RGB samples per textured row.
 *     3. Observer side: every camera k with an image, k != c, that sees f by texture_select's steps 1-3 (cfg.sel's z range, rule and
 *        positions, f's current flip): select's step-5 uv of f at cams[k], scaled to image k by rule 1, sampled as in 2.
 *     4. Clipping: a sample pair (I_k, I_c) is dropped when any of its six channel values is 0 or 255.
 *     5. Pair (k, c): per kept sample pair n += 1, S_k[ch] += I_k[ch], S_c[ch] += I_c[ch]; int64 sums, so exact and independent of
 *        order.  A pair exists where n >= 1; the list is in ascending (k, c).
 *     6. Normal equations per channel, K = n_cams unknowns: for each pair (a = k, b = c), A[a][a] += (S_a S_a / n) / sn2 + n / sg2,
 *        A[b][b] += (S_b S_b / n) / sn2 + n / sg2, A[a][b] and A[b][a] each -= (S_a S_b / n) / sn2, rhs[a] and rhs[b] each += n / sg2
 *        (sn2 = sigma_n sigma_n, sg2 = sigma_g sigma_g; products of int64 sums as doubles).  A camera in no pair takes the row g = 1
 *        (A = 1, rhs = 1).  A is symmetric positive definite with off-diagonal entries <= 0, so every gain is > 0.
 *     7. Solve: Jacobi-preconditioned conjugate gradients on the host from g = 1, dot products summed in camera order, the matrix
 *        applied as its diagonal then the pairs in list order; stop when |r| <= 1e-12 |rhs| or after max(100, 2 K) iterations.
 *   IMMESH_E_INVALID, nothing written: NULL h, cams, images, cfg or gains; n_cams < 1; on_device not 0 / 1; n_facets other than the
 *     live triangle count or > 0 with NULL rows; the bake's row checks (facet_cam in [-1, n_cams), finite uv); a textured row whose
 *     camera has a NULL image; a given image the bake refuses (sizes below 1, pitch below 3 width, a host image above max_image_bytes);
 *     a camera with an image that texture_select refuses; a cfg.sel texture_select refuses; sigma_n or sigma_g not finite or not > 0;
 *     max_pairs < 1; max_image_bytes < 0; a sharded handle.
 *   Not modelled: blending several views, local seam levelling, bias, gamma or vignetting, lens distortion.
 * immesh_texture_apply_gains: the corrected images, each channel out = min(255, floor(in g + 0.5)) in float64 with g = gains[k][ch].
 *   in [n] and out [n] images of equal sizes (out may be in: in place); an entry with NULL in data is skipped.  on_device 1: device
 *   memory of h's device, one kernel on h's stream, blocking; 0: host memory, a host loop.  The corrected images then go unchanged into
 *   texture_bake, render_textured and write_png.  IMMESH_E_INVALID, nothing written: NULL h, in, out or gains; n < 0; on_device not
 *   0 / 1; an entry with a NULL out, a size below 1, sizes that differ or a pitch below 3 width; a gain not finite or < 0. */
typedef struct {
    immesh_texture_config sel;   /* the select rule deciding whether an observer sees a facet; positions: the rows' own */
    double sigma_n, sigma_g;     /* Brown & Lowe's sigmas in 0-255 units: finite, > 0 (OpenCV's defaults: 10 and 0.1) */
    int64_t max_pairs;           /* >= 1: the capacity of the pair list */
    int64_t max_image_bytes;     /* host images: bytes of each of the two upload arenas (0: 512 MiB); must hold the largest image */
} immesh_texture_gains_config;
int immesh_mesh_texture_gains(immesh_mesh_t* h, const immesh_texture_camera* cams, int n_cams, const immesh_texture_image* images /*[n_cams]*/,
                              int on_device, const int32_t* facet_cam /*[n_facets]*/, const float* facet_uv /*[n_facets][6]*/, int64_t n_facets,
                              const immesh_texture_gains_config* cfg, double* gains /*[n_cams][3]*/, int32_t* pair_cam /*[max_pairs][2] or NULL*/,
                              int64_t* pair_sums /*[max_pairs][7] or NULL*/, int64_t* n_pairs /*or NULL*/, int64_t* counts /*[8] or NULL*/);
/* The phases of this thread's last immesh_mesh_texture_gains that reached the solve, in milliseconds: ms [3] = chosen samples (CUDA
 * events; with host images the uploads they wait for), observer passes (CUDA events; likewise), solve (host clock, read-back included). */
int immesh_mesh_texture_gains_stats(double* ms /*[3]*/);
int immesh_texture_apply_gains(immesh_mesh_t* h, const immesh_texture_image* in /*[n]*/, const immesh_texture_image* out /*[n]*/, int n, int on_device,
                               const double* gains /*[n][3]*/);
/* Voxel_mapping::kitti_log (src/voxel_mapping_common.cpp:43-70): one line "stamp tx ty tz qx qy qz qw\n" of the pose log in the KITTI camera
 * frame for the pose part (rot_end, pos_end) of a state vector.  Host-side only. */
int immesh_kitti_pose_line(const double* state /*[>=12]*/, double stamp, char* buf, int cap);
/* KD_TREE::Nearest_Search(point, k, ..., max_dist) (include/ikd-Tree/ikd_Tree.h:306) over the mesh vertices:
 * exact k nearest by float squared distance, ascending, ties by lower id; idx = -1 / d2 = inf when fewer exist. */
int immesh_knn(immesh_mesh_t* h, const float* query_xyz /*[nq][3]*/, int nq, int k, double max_dist, int32_t* idx /*[nq][k]*/,
               float* d2 /*[nq][k]*/);
/* per-frame work accounting used for the roofline arithmetic: [candidates, kNN candidates gathered, kNN queries,
 * dilated vertices, facets produced, voxels meshed, add-list entries, remove-list entries] */
int immesh_mesh_work_stats(immesh_mesh_t* h, int64_t* out /*[8]*/);
int immesh_mesh_last_timing(immesh_mesh_t* h, double* ms /*[4]: whole frame incl. H2D, append, per-voxel, push*/);

/* ---- front-end (SURVEY 8f-1): pcl::VoxelGrid centroid down-sampling of a scan on the device.  Replaces
 *   m_downSizeFilterSurf.setLeafSize(l, l, l); m_downSizeFilterSurf.setInputCloud(m_feats_undistort);
 *   m_downSizeFilterSurf.filter(*m_feats_down_body);      (src/voxel_mapping.cpp:1715, :1888-1889)
 * and the mesher's copy (src/ImMesh_mesh_reconstruction.cpp:335-338).  xyz: [n][3] floats like pcl::PointXYZI's x, y, z
 * (host pointer, or device pointer with on_device = 1).  Output: one centroid per occupied leaf, leaves in ascending
 * PCL cell index, [m][3]; it stays on the device (immesh_voxelgrid_device_points, valid until the next call on the
 * handle -- pass it to immesh_lio_step_async(..., on_device = 1)) and is copied to out_xyz when that is not NULL.
 * leaf_too_small mirrors PCL's "Leaf size is too small for the input dataset" branch (output = input, m = n). */
int immesh_voxelgrid_create(int max_points, immesh_voxelgrid_t** out);
int immesh_voxelgrid_destroy(immesh_voxelgrid_t* h);
int immesh_voxelgrid_filter(immesh_voxelgrid_t* h, const float* xyz, int n, int on_device, float leaf, float* out_xyz /*[n][3] or NULL*/,
                            int* m_out, int* leaf_too_small /*or NULL*/);
const float* immesh_voxelgrid_device_points(immesh_voxelgrid_t* h);
/* KITTI laser calibration (src/voxel_mapping.cpp:1844-1859, preprocess/calib_laser: the vertical angle of every return is raised
 * by 0.15 deg) + repacking: reads n points of `stride` floats (3: x y z; 4: x y z curvature, what immesh_imu_undistort emits),
 * applies the calibration when calib_laser != 0 and leaves the packed [n][3] cloud on the device (immesh_voxelgrid_input_points:
 * pass it to immesh_voxelgrid_filter with on_device = 1); copied to out_xyz when that is not NULL. */
int immesh_frontend_prepare(immesh_voxelgrid_t* h, const float* pts, int n, int stride, int on_device, int calib_laser, float* out_xyz /*[n][3] or NULL*/);
const float* immesh_voxelgrid_input_points(immesh_voxelgrid_t* h);
/* The whole front-end chain of one scan on the device, queued on the localization handle's stream without any host round trip:
 * [calibration] -> VoxelGrid down-sampling -> immesh_lio_step_async on the down-sampled cloud (its size stays on the device).
 * Replaces src/voxel_mapping.cpp:1844-1859 + :1888-1889 + lio_state_estimation + map_incremental_grow for the scan. */
int immesh_lio_step_async_raw(immesh_lio_t* lio, immesh_voxelgrid_t* h, const float* pts, int n, int stride, int on_device, int calib_laser, float leaf,
                              double dt, double cov_gyr, double cov_acc);

/* ---- depth cameras through the localization: the reference's preprocess/lidar_type 4 (L515; include/common_lib.h:66), whose
 * Preprocess::l515_handler (src/preprocess.cpp:234-275) turns the camera's cloud into the LiDAR scan of the imu_en: false loop
 * (Forward_without_imu, pcl::VoxelGrid, voxel_map_init / lio_state_estimation + map_incremental_grow, the mesher hand-off).
 * One depth image becomes one sensor-frame cloud, on the device:
 *   Sampling and validity: exactly those of immesh_depth_frame (stride, format, kind, z_min / z_max, the float64 arithmetic), with
 *     cam_R / cam_t mapping the camera to the sensor frame -- the frame the localization calls its LiDAR frame, which
 *     immesh_lio_config's ext_R / ext_T then map to the body as for any LiDAR.  Identity gives the camera-optical-frame cloud the
 *     L515 / RealSense driver publishes.
 *   point_filter_num (>= 1): the valid samples are numbered i = 0, 1, 2, ... in ascending pixel order (the order of the driver's
 *     unorganised cloud); sample i is kept iff i % point_filter_num == 0 (preprocess.cpp:250).
 *   blind (finite, >= 0), after the decimation: a kept point (x, y, z) (the float32 values) is dropped iff (double)r < blind * blind,
 *     r = (x*x + y*y) + z*z in float32 without FMA (preprocess.cpp:253-256).
 *   The survivors, in that order, are the cloud: float32 [n][3] in the VoxelGrid handle's input ring (immesh_voxelgrid_input_points),
 *     its count on the device (immesh_voxelgrid_input_count).  A host image is staged, sampled pixels only, through the handle's
 *     pinned staging; a device image is read in place at its pitch and must stay unchanged until the chain has run.
 * immesh_frontend_prepare_depth(vg, f, depth, on_device, point_filter_num, blind, out_xyz, cap, n_out): blocking; the cloud of one
 *   image, *n_out points, copied to out_xyz when cap >= *n_out (cap = 0: a count query; 0 < cap < *n_out: IMMESH_E_CAPACITY, nothing
 *   written).  The first frame's voxel_map_init is immesh_lio_predict + immesh_voxelmap_build on this cloud, as the reference's
 *   imu_en: false loop does (it meshes nothing for that frame).
 * immesh_lio_step_async_depth(lio, vg, f, depth, on_device, point_filter_num, blind, leaf, dt, cov_gyr, cov_acc): queued on the
 *   localization stream, no host synchronisation: the cloud -> pcl::VoxelGrid(leaf) (immesh_voxelgrid_filter with the count read on
 *   the device) -> predict + IESKF + map update (immesh_lio_step_async_dev_n).  The result equals immesh_lio_step_async_raw fed the
 *   same cloud.  A frame with no point left keeps what a zero device count does: the prediction is applied, the IESKF and the map
 *   update are skipped (the reference runs Forward_without_imu before its "No point" continue).  The scan feed records it with
 *   KIND = IMMESH_FEED_KIND_DEPTH; its full scan (registered = 2) is the filtered cloud.
 *   Hand the frame to the mesher after it with immesh_mesh_push_frame_from_lio_async_dev_n(mesh, lio,
 *   immesh_voxelgrid_input_points(vg), sampled pixels, immesh_voxelgrid_input_count(vg)).
 * immesh_voxelgrid_input_count(vg): device pointer to the count of the cloud immesh_voxelgrid_input_points returns when a depth entry
 *   point wrote it, else NULL; valid until that ring slot is reused (8 calls later).
 * immesh_mesh_push_frame_from_lio_async_dev_n(h, lio, d_body_xyz, n_max, d_n): immesh_mesh_push_frame_from_lio_async(h, lio,
 *   d_body_xyz, *d_n, 1) with the count read on the device (*d_n <= n_max): the frame's append_point_step and candidates are set
 *   there, with the rule of immesh_mesh_push_frame; the frame's grids cover n_max.  The frame feed records it with
 *   KIND = IMMESH_MFEED_KIND_FROM_LIO_ASYNC_DEV_N (N_POINTS, STEP: the device values).  *d_n == 0 adds nothing to the mesh.
 * Errors: the checks of immesh_depth_frame (IMMESH_E_INVALID), and IMMESH_E_INVALID for point_filter_num < 1, a negative or
 *   non-finite blind, leaf <= 0 or a sharded localization or mesh handle; IMMESH_E_CAPACITY when the sampled pixels exceed the
 *   VoxelGrid's max_points, or n_max > max_frame_points.  The down-sampled cloud must fit max_scan_points, as for
 *   immesh_lio_step_async_raw. */
int immesh_frontend_prepare_depth(immesh_voxelgrid_t* vg, const immesh_depth_frame* f, const void* depth, int on_device, int point_filter_num, double blind,
                                  float* out_xyz /*[cap][3] or NULL*/, int cap, int* n_out);
int immesh_lio_step_async_depth(immesh_lio_t* lio, immesh_voxelgrid_t* vg, const immesh_depth_frame* f, const void* depth, int on_device, int point_filter_num,
                                double blind, float leaf, double dt, double cov_gyr, double cov_acc);
const int* immesh_voxelgrid_input_count(immesh_voxelgrid_t* vg);
int immesh_mesh_push_frame_from_lio_async_dev_n(immesh_mesh_t* h, immesh_lio_t* lio, const float* d_body_xyz, int n_max, const int* d_n);

/* ---- point intensity through the front-end.  The reference keeps every PointType field through the front-end: the KITTI
 * calibration copies the whole point (src/voxel_mapping.cpp:1844-1859), and pcl::VoxelGrid (:1888-1889) runs with PCL's default
 * downsample_all_data_ = true, so each leaf's intensity is CentroidPoint's AccumulatorIntensity: the float sum over the leaf, in the
 * order of its x y z sums (ascending scan index here, see immesh_voxelgrid_filter), divided by (float)count.
 * The _i entry points take the caller's point records as `stride` floats per point: x y z in columns 0..2, the intensity in column
 * intensity_col (and, for the IMU chain, the time stamp, curvature in ms, in time_col) -- pcl::PointXYZINormal as it is: stride 12,
 * intensity 8, curvature 9.  stride <= 16, the columns distinct, >= 3 and < stride; host pointer, or device pointer with on_device.
 * Anything else: IMMESH_E_INVALID.  The intensity never enters what the localization or the mesher computes: the _i chains give the
 * state, map, effect rows and mesh of their plain counterparts fed the same x y z (and stamps).  The intensity buffers (and host
 * staging for wider records) are allocated by the first _i call on a handle.
 * A sharded localization handle: IMMESH_E_INVALID (the _i chains and immesh_lio_frontend_cloud run on a single GPU). */
/* immesh_voxelgrid_filter with intensity: same leaves, same order, bit-identical x y z; rows [m][4] = x y z intensity.  Non-finite
 * points are dropped with their intensity; in the leaf-too-small branch the output is the input, intensity included.
 * Replaces m_downSizeFilterSurf.filter(*m_feats_down_body) on PointXYZINormal clouds (src/voxel_mapping.cpp:1888-1889). */
int immesh_voxelgrid_filter_i(immesh_voxelgrid_t* h, const float* pts, int n, int stride, int intensity_col, int on_device, float leaf,
                              float* out_xyzi /*[m][4] or NULL*/, int* m_out, int* leaf_too_small /*or NULL*/);
/* immesh_lio_step_async_raw on point records, the intensity carried beside the clouds (src/voxel_mapping.cpp:1844-1859, :1888-1889):
 * immesh_voxelgrid_input_points(vg) stays the packed [n][3] scan (hand it to the mesher as after the plain chain); vg keeps its
 * intensity, and that of the down-sampled cloud, for immesh_lio_frontend_cloud. */
int immesh_lio_step_async_raw_i(immesh_lio_t* lio, immesh_voxelgrid_t* vg, const float* pts, int n, int stride, int intensity_col,
                                int on_device, int calib_laser, float leaf, double dt, double cov_gyr, double cov_acc);
/* publish_frame_world (src/voxel_mapping_common.cpp:595-614, pointBodyToWorld :121-131 with po.intensity = pi.intensity) from the
 * front-end's own clouds: dense != 0 -> the calibrated (undistorted, for the IMU chain time-sorted) full scan, m_feats_undistort;
 * else the down-sampled scan the last step localised, m_feats_down_body.  Rows [n][4] = world x y z, intensity
 * (IMMESH_SCAN_PUB_COLS) of points 0, point_skip, 2 point_skip, ..., transformed as immesh_lio_registered_cloud does, with the
 * handle's current state: the dense = 0 rows are those of immesh_lio_registered_cloud(lio, NULL, ...) with the intensity filled in.
 * transformLidar (:709-726) is the same arithmetic, so the viewer's current-scan points (g_eigen_vec_vec,
 * src/ImMesh_mesh_reconstruction.cpp:102-106) are the dense = 1, point_skip = 1 rows.  Blocking: waits for the work queued on lio;
 * the counts are read from the device.  *n_out > cap: IMMESH_E_CAPACITY with *n_out = rows needed (cap = 0: a count query).
 * IMMESH_E_INVALID, besides bad arguments, when the last step on lio did not come through immesh_lio_step_async_raw_i or branch 3 of
 * immesh_lio_step_async_imu_i with this vg (branches 1 and 2 publish nothing: the loop continues at src/voxel_mapping.cpp:1879,
 * :1903), or when vg has run any other call since. */
int immesh_lio_frontend_cloud(immesh_lio_t* lio, immesh_voxelgrid_t* vg, int dense, int point_skip, float* rows /*[cap][4]*/, int cap, int* n_out);

/* ---- front-end (SURVEY 8f-2): IMU forward propagation + per-point motion compensation on the device.  Replaces
 *   ImuProcess::UndistortPcl(lidar_meas, state_inout, pcl_out)            (src/IMU_Processing.cpp:755-958)
 * for the LiDAR-only flow (is_lidar_end == true).  The handle carries the ImuProcess members the function reads and writes
 * (cov_gyr / cov_acc / bias covariances :56-61, mean_acc from IMU_init :127-181, Lid_rot_to_IMU / Lid_offset_to_IMU :108-112,
 * last_imu_, last_lidar_end_time_, acc_s_last, angvel_last, lidar_meas.last_update_time); `state_inout` is the localization
 * handle's device-resident state: its rot / pos / vel are moved to the scan end and its 18x18 covariance is propagated
 * (F P F^T + Q per IMU interval).
 *   imu      : meas.imu of this scan, [n_imu][7] = stamp (s), angular_velocity xyz, linear_acceleration xyz
 *   pts_xyzt : [n][4] = x, y, z, curvature (ms since lidar_beg_time), float like pcl::PointXYZINormal; host pointer, or device
 *              pointer (16-byte aligned) with on_device = 1
 * Output: the scan sorted by time stamp (stable) and compensated into the scan-end frame, [n][4]; it stays on the device
 * (immesh_imu_device_points) and is copied to out_xyzt when that is not NULL.  Defined where the reference is not: points
 * with equal stamps keep their input order.  Work is queued on the localization handle's stream. */
typedef struct immesh_imu_config {
    double cov_gyr[3], cov_acc[3], cov_bias_gyr[3], cov_bias_acc[3];
    double mean_acc_norm;
    double lid_R[9]; /* row-major */
    double lid_T[3];
    int max_points;  /* capacity of one scan */
    int max_imu;     /* capacity of one IMU batch (<= 256) */
} immesh_imu_config;
int immesh_imu_create(const immesh_imu_config* cfg, immesh_imu_t** out);
int immesh_imu_destroy(immesh_imu_t* h);
/* seed the members IMU_init / the previous scan leave behind; acc_s_last / angvel_last may be NULL (zeros) */
int immesh_imu_reset(immesh_imu_t* h, const double* last_imu7, double last_lidar_end_time, double last_update_time, const double* acc_s_last,
                     const double* angvel_last);
int immesh_imu_undistort(immesh_imu_t* h, immesh_lio_t* lio, const double* imu, int n_imu, const float* pts_xyzt, int n, int on_device,
                         double lidar_beg_time, float* out_xyzt /*[n][4] or NULL*/);
const float* immesh_imu_device_points(immesh_imu_t* h);
/* IMUpose of the last call (Pose6D: offset_time, acc, gyr, vel, pos, rot = 22 doubles each); returns their number */
int immesh_imu_get_poses(immesh_imu_t* h, double* out, int cap_poses);

/* ---- the IMU-enabled scan loop (imu_en: true; config/avia.yaml, nclt.yaml, ntu.yaml): Voxel_mapping::service_LiDAR_update
 * (src/voxel_mapping.cpp:1820-1905 and on) with ImuProcess::Process2 (src/IMU_Processing.cpp:960-1006) and IMU_init, StatesGroup
 * version (src/IMU_Processing.cpp:188-232), as one queued call per scan.  Each scan takes exactly one branch:
 *   1 initialising (imu_need_init_): lidar_meas.last_update_time = pcl_end_time; on a non-empty batch IMU_init -- running means of the
 *     samples in the reference's order (on the host: the samples are host data), gravity = -mean_acc / |mean_acc| * 9.81, rot_end = I,
 *     bias_g = 0 written into the localization handle's state in stream order, last_imu_ = the batch's last sample; once
 *     init_iter_num (which counts samples) exceeds max_ini_count the phase ends and UndistortPcl scales the accelerations by |mean_acc|
 *     instead of immesh_imu_config::mean_acc_norm.  Nothing else: the reference's m_feats_undistort is empty and the loop continues.
 *   2 the first scan after it: UndistortPcl, [KITTI calibration], voxel_map_init from the full-resolution undistorted scan (queued:
 *     the build kernels of immesh_voxelmap_build read the calibrated scan on the device).  No IESKF, no map growth, no mesh frame.
 *   3 every later scan: UndistortPcl, [calibration], VoxelGrid(leaf), IESKF on the propagated state (no Forward_without_imu),
 *     map_incremental_grow -- immesh_lio_step_async_raw on the undistorted scan.  Hand the frame to the mesher after it with
 *       immesh_mesh_push_frame_from_lio_async(mesh, lio, immesh_voxelgrid_input_points(vg), n, 1)
 *     before the next call on vg (the input ring of vg keeps the packed scan for the frames still in flight).
 * *branch_out = the branch taken.  It depends on sample counts and the first-map flag only, so the host knows it without waiting.  The
 * call waits for the device only on a busy staging slot (immesh_host_wait_ms, localization handle); immesh_lio_wait drains it.
 * The first-map flag is set by branch 2 and kept across immesh_imu_init_begin (the reference's m_init_map survives its reset).
 * Defined where the reference is not: last_lidar_end_time_ (src/IMU_Processing.h:146) has no initialiser and nothing sets it before
 * the first UndistortPcl: it is 0.0 here (what the zero-filled heap the reference runs on gives).
 * imu: [n_imu][7] host array (stamp, gyr xyz, acc xyz); pts_xyzt: [n][4] as for immesh_imu_undistort (host, or device with on_device).
 * Errors, returned before anything is queued or any counter moves: n_imu > max_imu, n > the IMU or VoxelGrid handle's max_points, or
 * n > the localization handle's max_scan_points (the map is built from the whole scan, and a scan the VoxelGrid passes through reaches
 * the step whole): IMMESH_E_CAPACITY; a sharded localization handle: IMMESH_E_INVALID. */
/* Enter branch 1.  The first call on a handle starts from a fresh ImuProcess (b_first_frame_: the first batch seeds the means; zero
 * last_imu_, acc_s_last, angvel_last).  A later call is the loop's reset (m_flg_reset -> Reset(), src/voxel_mapping.cpp:1791-1796):
 * b_first_frame_ stays false, so the means restart from mean_acc = (0, 0, -1), mean_gyr = 0 with init_iter_num = 1; last_imu_ and
 * angvel_last are zeroed, acc_s_last and last_lidar_end_time_ kept.  A handle that never calls it has no initialisation phase:
 * immesh_lio_step_async_imu starts at branch 2 with the configured mean_acc_norm (the caller-initialised flow).
 * max_ini_count = MAX_INI_COUNT (mapping/imu_int_frame, 3 by default). */
int immesh_imu_init_begin(immesh_imu_t* h, int max_ini_count);
int immesh_lio_step_async_imu(immesh_lio_t* lio, immesh_imu_t* imu_h, immesh_voxelgrid_t* vg, const double* imu /*[n_imu][7]*/, int n_imu,
                              const float* pts_xyzt /*[n][4]*/, int n, int on_device, double lidar_beg_time, int calib_laser, float leaf,
                              int* branch_out /*or NULL*/);
/* immesh_lio_step_async_imu on point records (see immesh_voxelgrid_filter_i): lidar_meas.lidar as it is, the time stamp in time_col.
 * UndistortPcl sorts and compensates whole PointType records (src/IMU_Processing.cpp:784, time_list :48): the intensity follows its
 * point through the same stable time sort, then through the calibration and the VoxelGrid as in immesh_lio_step_async_raw_i.
 * Branches, state, map and mesh hand-off are those of immesh_lio_step_async_imu fed the same x y z t. */
int immesh_lio_step_async_imu_i(immesh_lio_t* lio, immesh_imu_t* imu_h, immesh_voxelgrid_t* vg, const double* imu /*[n_imu][7]*/, int n_imu,
                                const float* pts, int n, int stride, int time_col, int intensity_col, int on_device,
                                double lidar_beg_time, int calib_laser, float leaf, int* branch_out /*or NULL*/);

/* ---- the IMU-enabled loop on depth frames (L515, D435i, Azure Kinect with imu_en: true): immesh_lio_step_async_imu fed the depth
 * frame's cloud of immesh_lio_step_async_depth, one queued call per frame, with every decision the reference makes from the cloud made on
 * the device.  Nothing is read back: the cloud's count exists only on the device, so the host queues the same launches for every frame
 * and each kernel returns early unless its branch is the one the device took.
 *   Cloud: that of immesh_frontend_prepare_depth (f, depth, on_device, point_filter_num, blind), as x y z t records with t = 0
 *     (Preprocess::l515_handler sets curvature = 0, src/preprocess.cpp:270).  lidar_beg_time = frame_time, so pcl_end_time = frame_time.
 *     The stable time sort of all-equal stamps is the identity.  The KITTI calibration does not apply to depth frames (calib_laser = 0).
 *   Drop (sync_packages, src/voxel_mapping_common.cpp:393-400): a cloud of <= 1 point is dropped -- no state, last_update_time or
 *     initialisation change -- and the frame's IMU samples are carried on the device: the next frame's meas.imu is the carried samples,
 *     then its own, in order.  Carried + own samples beyond max_imu: the frame is dropped and its own samples discarded; the scan feed's
 *     ERR holds the flag from that frame on, and immesh_lio_wait (and every blocking localization call) returns IMMESH_E_CAPACITY from
 *     then on: the flag joins the handle's never-reset error word, like a pool overflow.  An overflow does not heal itself: the carry is
 *     only consumed by a kept frame, and while carry + a frame's samples exceed max_imu every frame is dropped -- size max_imu for the
 *     longest run of dropped frames, or restart with immesh_imu_init_begin (which discards the carry).
 *   Otherwise the branch of immesh_lio_step_async_imu, from the device's phase (Process2, src/IMU_Processing.cpp:960-1006;
 *     src/voxel_mapping.cpp:1820-1905):
 *     1 initialising: IMU_init (:188-232) on the device, the same code as the host chain's (running means in sample order, no FMA),
 *       the init-end test init_iter_num > max_ini_count and |mean_acc| on the device; last_update_time = frame_time.
 *     2 the first frame after it: UndistortPcl, then voxel_map_init from the whole undistorted cloud.
 *     3 every later frame: UndistortPcl, VoxelGrid(leaf), IESKF on the propagated state and the map update.
 *   Scan feed: one record per call, KIND = IMMESH_FEED_KIND_DEPTH_IMU, BRANCH = 1, 2, 3 or IMMESH_FEED_BRANCH_DROPPED (header and state
 *     only unless 3).  Branch 3's full scan (registered = 2) is the undistorted cloud.
 *   Mesh hand-off, after every call: immesh_mesh_push_frame_from_lio_async_dev_n(mesh, lio, immesh_voxelgrid_input_points(vg), sampled
 *     pixels, immesh_voxelgrid_input_count(vg)).  The count is the undistorted cloud's in branch 3 and 0 otherwise.  The reference hands
 *     off nothing for the other frames; here they are mesh frames that add nothing, and the mesh frame feed shows them with N_POINTS = 0.
 * The call waits for the device only on a busy staging slot (immesh_host_wait_ms counts it: the IMU batch's and the localization's
 *   slots -- two per call, the build's and the step's -- and, for a host image, the VoxelGrid's image staging) and, with pool growth on,
 *   where immesh_lio_config's growth needs a drain as on every chain.  Its step replays the captured launch sequence of
 *   immesh_lio_step_async_dev_n; the direct launches (profiling on) give the same results.
 * Input and pose rings: one slot of each per call, as on the other chains -- the cloud is unprojected into an input-ring slot and the
 *   undistorted cloud written back into it, and the build shares the step's scan index.
 * Handle rules: once this entry point has run on an IMU handle, the handle's phase, first-map flag and carry live on the device;
 *   immesh_lio_step_async_imu[_i] on it then returns IMMESH_E_INVALID, as this one does on a handle they have run on.
 *   immesh_imu_init_begin restarts the phase as documented there (the carried samples are discarded: they belong before the reset).
 * Errors, returned before anything is queued: those of immesh_lio_step_async_depth, IMMESH_E_CAPACITY for n_imu > max_imu, or sampled
 *   pixels beyond the IMU handle's max_points or the localization handle's max_scan_points; IMMESH_E_INVALID for a sharded handle.
 *   Exception: a pool growth the localization's build or step then needs can still fail (IMMESH_E_CAPACITY / IMMESH_E_CUDA) after the
 *   frame's decision is queued: the device phase and carry have then taken the frame without its step.
 * immesh_imu_depth_chain_state (blocking): out = [calls, dropped, branch-1, branch-2, branch-3 frames, carried samples now, carry
 *   overflows, initialisation finished (0/1)]. */
int immesh_lio_step_async_depth_imu(immesh_lio_t* lio, immesh_imu_t* imu_h, immesh_voxelgrid_t* vg, const double* imu /*[n_imu][7]*/, int n_imu,
                                    const immesh_depth_frame* f, const void* depth, int on_device, int point_filter_num, double blind,
                                    double frame_time, float leaf);
int immesh_imu_depth_chain_state(immesh_imu_t* h, int64_t out[8]);

/* optional per-kernel CUDA-event profiler (off by default) and launch accounting, process-wide */
int immesh_profile_enable(int on);   /* 0 off, 1 per-kernel totals, 2 totals + timeline */
int immesh_profile_timeline(char* buf, int cap); /* "kernel t0_ms t1_ms\n" per launch; returns bytes needed */
int immesh_profile_reset(void);
int immesh_profile_report(char* buf, int cap); /* "kernel ms launches\n" lines; returns bytes needed */
long long immesh_launch_count(void);
/* CUDA-graph replay accounting of the pipelined entry points: [lio captures, lio replays, lio failures, mesh captures,
 * mesh replays, mesh failures]; either handle may be NULL */
int immesh_graph_stats(immesh_lio_t* lio, immesh_mesh_t* mesh, int64_t* out /*[6]*/);
/* programmatic dependent-launch edges of the captured graphs: [lio, mesh] (0 while a handle has no captured graph); either
 * handle may be NULL */
int immesh_graph_pdl_edges(immesh_lio_t* lio, immesh_mesh_t* mesh, int64_t* out /*[2]*/);

const char* immesh_last_error(void);
const char* immesh_version(void);

#ifdef __cplusplus
}
#endif
#endif /* IMMESH_B200_H_ */
