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
 * device scan must still hold it), intensity 0 -- the device VoxelGrid does not carry intensity (PCL's averages it); n, stride,
 * intensity_col and on_device are then ignored.
 * point_skip <= 0 (the reference would loop forever), stride < 3 or intensity_col >= stride: IMMESH_E_INVALID. */
int immesh_lio_registered_cloud(immesh_lio_t* h, const float* pts, int n, int stride, int intensity_col, int on_device,
                                int point_skip, float* rows /*[cap][4]*/, int cap, int* n_out);

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
/* host time (ms) the queueing calls spent blocked on a busy staging slot (back-pressure from the device, not work) since the
 * last call: out[0] localization handle, out[1] meshing handle; either handle may be NULL */
int immesh_host_wait_ms(immesh_lio_t* lio, immesh_mesh_t* h, double* out /*[2]*/);
/* CUDA-event time (ms) of everything queued on both handles between the two marks */
int immesh_pipeline_mark_begin(immesh_lio_t* lio);
int immesh_pipeline_mark_end(immesh_lio_t* lio, immesh_mesh_t* h, double* ms);
/* counts: [n_vertices, n_live_triangles, frame_new_vertices, frame_voxels_meshed, frame_added, frame_removed, n_voxels, n_activated] */
int immesh_mesh_counts(immesh_mesh_t* h, int64_t* out /*[8]*/);
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

/* optional per-kernel CUDA-event profiler (off by default) and launch accounting, process-wide */
int immesh_profile_enable(int on);   /* 0 off, 1 per-kernel totals, 2 totals + timeline */
int immesh_profile_timeline(char* buf, int cap); /* "kernel t0_ms t1_ms\n" per launch; returns bytes needed */
int immesh_profile_reset(void);
int immesh_profile_report(char* buf, int cap); /* "kernel ms launches\n" lines; returns bytes needed */
long long immesh_launch_count(void);
/* CUDA-graph replay accounting of the pipelined entry points: [lio captures, lio replays, lio failures, mesh captures,
 * mesh replays, mesh failures]; either handle may be NULL */
int immesh_graph_stats(immesh_lio_t* lio, immesh_mesh_t* mesh, int64_t* out /*[6]*/);

const char* immesh_last_error(void);
const char* immesh_version(void);

#ifdef __cplusplus
}
#endif
#endif /* IMMESH_B200_H_ */
