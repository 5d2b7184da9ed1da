/*
 * ovn_b200.h -- C ABI of the Hopper-native (sm_90a) OverlapNet inference hot path (libovn_b200.so).
 *
 * The reference (PRBonn/OverlapNet) has no FFI / plugin interface: its boundary is the Python
 * class `Infer` (src/two_heads/infer.py:22-265) plus the NumPy preprocessing functions
 * (src/utils/utils.py:59-186).  This header is the native boundary a maintainer binds underneath
 * those Python entry points (ctypes stub in INTEGRATION.md); every function names the reference
 * code it replaces.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no C++/torch types.
 *   - Pointers named d_* are DEVICE pointers, h_* are HOST pointers.
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).  Device-pointer
 *     entry points are asynchronous on that stream and never synchronise the host; host-buffer
 *     entry points (suffix _host) copy in/out and return after the result is on the host.
 *   - Every function returns an ovn_status (0 = OK, negative = error); no exception crosses the ABI.
 *     ovn_last_error(h) gives the message for the last failure on that handle.
 *   - A handle owns the packed weights and all workspaces, is bound to the CUDA device that was
 *     current at ovn_create(), and is NOT thread-safe (like `Infer`: infer.py keeps a mutable
 *     feature bank, SURVEY 8b "Threading").
 *   - Feature volumes cross the ABI as float32 [n][W_out=360][128] (what
 *     Infer.create_feature_volumes returns, infer.py:240-265, with the singleton H axis dropped).
 *   - ovn_copy_heads_stage reads back the intermediate stages of the tensor-core heads and ovn_leg_stage
 *     one layer of the tensor-core leg (tests and diagnostics only; the heads and leg calls do no extra
 *     work for them).  ovn_set_train_stop / ovn_copy_train_stage do the same for the training step.
 */
#ifndef OVN_B200_H_
#define OVN_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OVN_ABI_VERSION 1

typedef enum ovn_status {
  OVN_OK = 0,
  OVN_ERR_INVALID_ARG = -1,    /* NULL pointer, bad size, bad enum */
  OVN_ERR_BAD_CONFIG = -2,     /* unsupported model wiring (config/network.yml:64-82) */
  OVN_ERR_WEIGHTS = -3,        /* unknown layer name / wrong shape / weights not finalised */
  OVN_ERR_CUDA = -4,           /* a CUDA runtime call failed; see ovn_last_error */
  OVN_ERR_NO_DEVICE = -5,      /* no sm_90 device: the library has NO CPU fallback */
  OVN_ERR_CAPACITY = -6        /* batch larger than the workspace reserved at ovn_create */
} ovn_status;

/* Arithmetic of the network kernels. */
typedef enum ovn_precision {
  OVN_PREC_FP32 = 0,           /* fp32 SIMT kernels (verification path) */
  OVN_PREC_F16_TC = 1          /* fp16 (hi/lo split) operands, fp32 accumulate, tensor cores */
} ovn_precision;

/*
 * Model + projection configuration.  Mirrors the keys Infer.__init__ reads from
 * config/network.yml (infer.py:32-93) and the defaults of range_projection (utils.py:59).
 */
typedef struct ovn_config {
  int32_t abi_version;            /* must be OVN_ABI_VERSION */
  /* range projection, utils.py:59 */
  int32_t proj_H, proj_W;         /* 64, 900 (network.yml:75 inputShape) */
  float   fov_up_deg, fov_down_deg; /* 3.0, -25.0 */
  float   max_range;              /* 50.0 */
  /* input cues, network.yml:20-24, channel order ImagePairOverlapOrientationSequence.py:143-207 */
  int32_t use_depth;              /* 1 channel  */
  int32_t use_normals;            /* 3 channels */
  int32_t n_prob_channels;        /* 0, 3 (pca) or 20 */
  int32_t use_intensity;          /* 1 channel  */
  /* leg, generateNet.py:119-219 / network.yml:70-82 */
  int32_t strides_layer1[2];      /* (2,2) */
  int32_t additional_unsymmetric_layer3a; /* 1 */
  int32_t leg_output_width;       /* 360 */
  /* overlap head, generateNet.py:88-89 */
  int32_t conv1size;              /* 15 */
  /* execution */
  int32_t precision;              /* ovn_precision */
  int32_t max_batch_scans;        /* workspace: scans per ovn_leg_forward / ovn_project_batch call */
  int32_t max_batch_pairs;        /* workspace: pairs per ovn_heads_forward call */
} ovn_config;

typedef struct ovn_handle ovn_handle;

/* ---- lifetime -------------------------------------------------------------------------- */
void        ovn_default_config(ovn_config* cfg);            /* network.yml geo-only defaults */
int         ovn_create(const ovn_config* cfg, ovn_handle** out);   /* replaces Infer.__init__ model build, infer.py:86-111 */
int         ovn_destroy(ovn_handle* h);
const char* ovn_last_error(const ovn_handle* h);
const char* ovn_status_string(int status);
int         ovn_abi_version(void);
int         ovn_input_channels(const ovn_handle* h);        /* infer.py:61-73 */
int         ovn_feature_width(const ovn_handle* h);         /* 360 */
int         ovn_feature_channels(const ovn_handle* h);      /* 128 */
/* Number of kernels this handle has launched so far (bench.py's gpu_launches). */
int64_t     ovn_launch_count(const ovn_handle* h);

/* ---- per-kernel device timing (bench.py roofline): CUDA events recorded around the named kernels
 * on the launching stream while enabled.  ovn_profile_read synchronises the device, returns the
 * accumulated milliseconds / launch count since the last read and resets them.  Names:
 * "delta_conv1", "conv2", "conv3", "corr", "project_scatter", "project_gather", "leg", "gather_rows",
 * "rows_topk", "pgo_graphs", "render_scatter", "render_gather", "surfel_build", "surfel_scatter",
 * "surfel_gather". */
int ovn_profile_enable(ovn_handle* h, int on);
int ovn_profile_read(ovn_handle* h, const char* kernel, double* total_ms, int64_t* launches);

/* ---- weights: replaces load_weights(by_name=True), infer.py:117-120 ----------------------- */
/* kernel: Keras layout, conv (kh,kw,cin,cout) / dense (in,out), float32 host memory; bias (cout).
 * Layer names: s_conv1..s_conv10 (+s_conv3a), c_conv1..c_conv3, overlap_output
 * (generateNet.py:99-114,162-214). */
int ovn_set_weights(ovn_handle* h, const char* layer_name,
                    const float* h_kernel, const int64_t* kernel_dims, int32_t kernel_ndim,
                    const float* h_bias, int64_t bias_len);
int ovn_finalize_weights(ovn_handle* h);   /* pack + upload; every layer must have been set */

/* ---- stage 1: range projection (utils.py:59-134) ------------------------------------------ */
/* d_points: [n_total][4] float32 x,y,z,intensity of `n_scans` clouds back to back;
 * d_offsets: [n_scans+1] int64 point offsets (device).  Outputs are optional (NULL = skip):
 *   d_range [n][H][W] f32, d_vertex [n][H][W][4] f32, d_intensity [n][H][W] f32,
 *   d_idx [n][H][W] i32 (index into the FILTERED cloud, utils.py:76,117-118).
 * max_range < 0 selects the handle's configured max_range; +inf is allowed
 * (gen_semantic_data.py:39). */
int ovn_project_batch(ovn_handle* h, const float* d_points, const int64_t* d_offsets, int32_t n_scans,
                      int64_t n_points_total, float max_range,
                      float* d_range, float* d_vertex, float* d_intensity, int32_t* d_idx,
                      void* stream);

/* ---- stage 1b: normal map (utils.py:137-175) ---------------------------------------------- */
int ovn_normals_batch(ovn_handle* h, const float* d_range, const float* d_vertex, int32_t n_scans,
                      float* d_normal /* [n][H][W][3] */, void* stream);

/* ---- stage 1c: semantic gather (gen_semantic_data.py:41-46, incl. the filtered-index quirk) */
int ovn_semantic_batch(ovn_handle* h, const int32_t* d_idx, const float* d_probs,
                       const int64_t* d_offsets, int32_t n_scans, int32_t n_classes,
                       float* d_out /* [n][H][W][n_classes] */, void* stream);

/* ---- ground-truth generator (com_overlap_yaw.py:10-68; SURVEY 8f-2) ------------------------- */
/* Float32 range images [n][H][W] of scans moved into the current frame: every point (x, y, z, 1)
 * is multiplied, in float64, by d_pose_ref[scan] and then by d_pose_cur_inv (row-major 4x4, either
 * may be NULL = identity; com_overlap_yaw.py:39-40) and projected by range_projection evaluated in
 * FLOAT64 (the reference's load_vertex builds a float64 array, utils.py:218-231; bins utils.py:75-104),
 * nearest point per pixel, depth rounded to float32 on store, -1 where empty (utils.py:120,129).
 * max_range < 0 selects the handle's configured max_range. */
int ovn_gt_range_batch(ovn_handle* h, const float* d_points, const int64_t* d_offsets, int32_t n_scans,
                       int64_t n_points_total, const double* d_pose_ref /* [n][16] */,
                       const double* d_pose_cur_inv /* [16] */, float max_range,
                       float* d_range /* [n][H][W] */, void* stream);

/* d_counts[b] = #{pixels: ref_b > 0 and |ref_b - cur| < 1} for b < n_scans (com_overlap_yaw.py:44-45,
 * float32 arithmetic); d_counts[n_scans] = #{cur > 0} = the reference's valid_num (:31-32). */
int ovn_gt_overlap_count(ovn_handle* h, const float* d_ref_ranges /* [n][H][W] */,
                         const float* d_cur_range /* [H][W] */, int32_t n_scans,
                         int32_t* d_counts /* [n_scans + 1] */, void* stream);

/* ---- ground truth for every frame pair (demo4_gen_gt_files.py over a whole sequence) -------------
 * The clouds stay resident on the device.  d_radius[b] = max ||p|| of scan b in float64 (0 if empty);
 * compute it once per upload for ovn_gt_pairs_count. */
int ovn_gt_scan_radius(ovn_handle* h, const float* d_points, const int64_t* d_offsets /* [n+1] */,
                       int32_t n_scans, double* d_radius /* [n] */, void* stream);

/* d_counts[f * ld_counts + r] = what ovn_gt_range_batch(reference scan r, d_pose_ref[r], d_pose_cur_inv[f])
 * followed by ovn_gt_overlap_count(..., d_cur_range[f]) gives, bit for bit, for every current frame f < n_cur
 * and reference scan r < n_ref.  Reference scan r is the points [h_offsets[r], h_offsets[r+1]) of d_points
 * (the offsets are read on the host).  d_cur_range [n_cur][H][W]: the frames' untransformed images
 * (ovn_gt_range_batch without poses).  Frames x references are processed in tiles of tile_cur x tile_ref
 * pairs (<= 0: defaults sized so that the tile's key images stay in L2; more than 32 x 64 is
 * OVN_ERR_CAPACITY); the counts do not depend on the tiling.  A pair whose every point provably lies at or
 * beyond max_range (||t_rel|| - s(R_rel) d_radius[r] - eps >= max_range, DESIGN.md section 4) is skipped with
 * count 0; *d_n_pruned (device, may be NULL) receives their number.  max_range < 0 selects the handle's.
 * The key-image workspace is allocated by the first call. */
int ovn_gt_pairs_count(ovn_handle* h, const float* d_points, const int64_t* h_offsets /* [n_ref+1], host */,
                       int32_t n_ref, const double* d_pose_ref /* [n_ref][16] */, const double* d_radius /* [n_ref] */,
                       const float* d_cur_range /* [n_cur][H][W] */, const double* d_pose_cur_inv /* [n_cur][16] */,
                       int32_t n_cur, float max_range, int32_t tile_cur, int32_t tile_ref,
                       int32_t* d_counts /* [n_cur][ld_counts] */, int64_t ld_counts, int64_t* d_n_pruned,
                       void* stream);

/* ---- stage 1d: fused raw cloud -> packed network input ------------------------------------- */
/* Projection + normals + channel packing (ImagePairOverlapOrientationSequence.py:130-207) in one
 * pass; d_probs may be NULL when n_prob_channels == 0.  d_input: [n][H][W][C] float32. */
int ovn_preprocess_batch(ovn_handle* h, const float* d_points, const int64_t* d_offsets,
                         int32_t n_scans, int64_t n_points_total, const float* d_probs,
                         float* d_input, void* stream);

/* The fused path with every cue as the reference's cue files give it.  Depth, normals and intensity are
 * gen_depth/normal/intensity_data.py's (the configured max_range); the class probabilities are
 * gen_semantic_data.py:33-46's: projected with max_range = inf (:39), and the probabilities of each pixel's
 * nearest point are read from the scan's RAW probability array at that point's index among the points with
 * 0 < depth < inf (:41-46, the reference's filtered-index quirk).  So d_input equals ovn_pack_input of those
 * four cues bit for bit, from one scatter (two key images per scan) and one gather.  d_probs:
 * [n_points_total][n_prob_channels] float32 (device), required iff n_prob_channels > 0, NULL otherwise
 * (OVN_ERR_INVALID_ARG); on a handle without probability channels this is ovn_preprocess_batch. */
int ovn_preprocess_cues_batch(ovn_handle* h, const float* d_points, const int64_t* d_offsets,
                              int32_t n_scans, int64_t n_points_total, const float* d_probs,
                              float* d_input, void* stream);

/* ---- stage 1e: virtual scans rendered from resident clouds (DESIGN.md sections 4 and 7) -------------
 * n_virtual images, each from a list of entries: image v takes the entries [h_entry_offsets[v],
 * h_entry_offsets[v+1]) (h_entry_offsets[0] = 0).  Entry e is the resident cloud h_entry_cloud[e], the points
 * [h_offsets[c], h_offsets[c+1]) of d_points ([n][4] float32 back to back, as for ovn_project_batch; h_offsets
 * is read on the host), moved by the row-major float64 pose h_entry_pose[e] ([16], bottom row 0 0 0 1; callers
 * compose it as T_v^-1 T_k).  Each point becomes q = fl32(M (x, y, z, 1)): every coordinate is
 * ((M_i0 x + M_i1 y) + M_i2 z) + M_i3 in float64, each product and sum rounded once (no FMA), then rounded to
 * float32; the intensity is kept.  Image v is then, bit for bit, what ovn_project_batch gives for the cloud that
 * concatenates the entries' transformed clouds in entry order, at the handle's geometry and max_range (< 0: the
 * handle's): the nearest point wins, the lower concatenated index on exact ties.  d_winner [n][H][W] int32 is
 * the winner's index in that concatenated cloud (not in the filtered one, unlike d_idx), -1 where empty; an
 * image with no entries is all -1.  Outputs may be NULL.
 * Caveat: with M = I a coordinate -0 becomes +0 (-0 + 0 = +0), and a point with y = -0 and x < 0 moves from
 * column W-1 to column 0; so an identity entry equals ovn_project_batch only for clouds without negative zeros.
 * The host tables are read and checked before anything is launched: decreasing offsets, h_entry_offsets[0] != 0,
 * a cloud index outside [0, n_clouds), a pose that is not finite or whose bottom row is not 0 0 0 1, and an
 * image whose concatenated points reach 2^32 (the key's index field; d_winner holds the index's low 32 bits)
 * are OVN_ERR_INVALID_ARG, with the handle still usable.  n_virtual > max_batch_scans is OVN_ERR_CAPACITY.
 * The entry table goes through a handle-owned device buffer, grown on use.  Profiled as "render_scatter" and
 * "render_gather". */
int ovn_render_batch(ovn_handle* h, const float* d_points, const int64_t* h_offsets /* [n_clouds+1] */,
                     int32_t n_clouds, int32_t n_virtual, const int64_t* h_entry_offsets /* [n_virtual+1] */,
                     const int32_t* h_entry_cloud /* [n_entries] */, const double* h_entry_pose /* [n_entries][16] */,
                     float max_range, float* d_range, float* d_vertex, float* d_intensity,
                     int32_t* d_winner /* [n][H][W] */, void* stream);

/* The render packed as ovn_preprocess_batch packs a projection: d_input [n_virtual][H][W][C] at the handle's
 * max_range.  OVN_ERR_BAD_CONFIG on a handle with probability channels: renders carry none. */
int ovn_render_preprocess_batch(ovn_handle* h, const float* d_points, const int64_t* h_offsets, int32_t n_clouds,
                                int32_t n_virtual, const int64_t* h_entry_offsets, const int32_t* h_entry_cloud,
                                const double* h_entry_pose, float* d_input, void* stream);

/* ---- stage 1f: virtual scans rendered from surfels (DESIGN.md sections 4 and 7, "Surfel renders") -------------
 * A keyframe's surfels are its projection's pixels (the handle's geometry and max_range): slot y W + x of its
 * [H][W][8] float32 bank holds (cx, cy, cz, r, nx, ny, nz, intensity), c the pixel's vertex, n its normal (the
 * sensor-facing -c / |c| where gen_normal_map leaves the (-1, -1, -1) fill) and r = fl32(((kappa d) delta) /
 * max(|n.c| / d, c_min)) in float64, d the pixel's range and delta = max(2 pi / W, fov / H).  An empty pixel is an
 * all-zero slot (r = 0, never drawn).  The defaults (kappa 1, c_min 0.5, max_splat 8) come from a synthetic street
 * study, not from KITTI. */
#define OVN_SURFEL_MAX_SPLAT_LIMIT 32
typedef struct ovn_surfel_params {
  double kappa;           /* radius scale, > 0 */
  double c_min;           /* the least |cos| between a normal and its pixel's ray in the radius, (0, 1] */
  int32_t max_splat;      /* a surfel is tested on the pixels within max_splat rows and columns of its centre, 0 .. 32 */
} ovn_surfel_params;
void ovn_surfel_default_params(ovn_surfel_params* p);
/* The surfel banks of n_clouds clouds (d_points / d_offsets as for ovn_project_batch), d_surfels [n][H][W][8].
 * Profiled as "project_scatter", "project_gather" and "surfel_build".  n_clouds > max_batch_scans is
 * OVN_ERR_CAPACITY. */
int ovn_surfels_batch(ovn_handle* h, const float* d_points, const int64_t* d_offsets, int32_t n_clouds,
                      int64_t n_points_total, const ovn_surfel_params* params, float* d_surfels, void* stream);
/* n_virtual images z-buffered from surfel banks, with the entry tables of ovn_render_batch (entry e: bank
 * h_entry_cloud[e] of d_surfels [n_clouds][H][W][8], moved by h_entry_pose[e]).  d_rays [H][W][3] float64: the
 * unit directions of the pixel centres (virtual_map.pixel_rays).  Per surfel, q = M (c, 1) in mat4_apply's order and
 * m = R n, in float64 without contraction; it is culled when |q| - r >= max_range or fl32(q) has depth 0, and tested
 * on the pixels within max_splat rows (clipped) and columns (circular) of fl32(q)'s projection pixel.  At pixel ray u:
 * t = (m.q) / (m.u), drawn when |m.u| > 1e-6, t > 0, fl32(t) < max_range and |t u - q|^2 <= r^2.  The key is
 * float_bits(fl32(t)) << 32 | (entry ordinal in the image * H W + slot), so the nearest hit wins, then the lowest
 * entry, then the lowest slot.  The gather gives range fl32(t), vertex fl32(t u), the surfel's intensity, and
 * d_winner = the key's index (its low 32 bits as int32), -1 where empty.  So each image is what the projection gives
 * for a scan whose points are the hit points.  max_range < 0 selects the handle's.  The host tables get
 * ovn_render_batch's checks and codes; an image of 2^32 / (H W) entries or more, a NULL d_surfels or d_rays with
 * entries, and bad parameters (kappa <= 0, a non-finite value, c_min outside (0, 1], max_splat outside [0, 32]) are
 * OVN_ERR_INVALID_ARG; n_virtual > max_batch_scans is OVN_ERR_CAPACITY.  Profiled as "surfel_scatter" and
 * "surfel_gather". */
int ovn_render_surfels_batch(ovn_handle* h, const float* d_surfels, int32_t n_clouds, const double* d_rays,
                             int32_t n_virtual, const int64_t* h_entry_offsets /* [n_virtual+1] */,
                             const int32_t* h_entry_cloud, const double* h_entry_pose /* [n_entries][16] */,
                             const ovn_surfel_params* params, float max_range, float* d_range, float* d_vertex,
                             float* d_intensity, int32_t* d_winner, void* stream);
/* The surfel render packed as ovn_preprocess_batch packs a projection: d_input [n_virtual][H][W][C] at the handle's
 * max_range.  OVN_ERR_BAD_CONFIG on a handle with probability channels: renders carry none. */
int ovn_render_surfels_preprocess_batch(ovn_handle* h, const float* d_surfels, int32_t n_clouds, const double* d_rays,
                                        int32_t n_virtual, const int64_t* h_entry_offsets,
                                        const int32_t* h_entry_cloud, const double* h_entry_pose,
                                        const ovn_surfel_params* params, float* d_input, void* stream);

/* Pack separately computed cue images into the NHWC network input (same channel order). */
int ovn_pack_input(ovn_handle* h, const float* d_depth, const float* d_normal, const float* d_prob,
                   const float* d_intensity, int32_t n_scans, float* d_input, void* stream);

/* ---- stage 2: leg encoder (generateNet.py:161-217; Infer.create_feature_volumes) ----------- */
/* d_input [n][H][W][C] f32 -> d_fv [n][360][128] f32. */
int ovn_leg_forward(ovn_handle* h, const float* d_input, int32_t n_scans, float* d_fv, void* stream);

/* ---- stage 3: heads (generateNet.py:15-116, 327-354; readout infer.py:157-158) ------------- */
/* Pair p uses LEFT = d_bank[left_idx[p]], RIGHT = d_bank[right_idx[p]]
 * (ImagePairOverlapSequenceFeatureVolume.py:44-45).  Outputs: d_overlap [n] f32,
 * d_yaw [n] i32 = 180 - argmax(corr) (first maximum; 180 at every leg_output_width, as infer.py:158),
 * d_corr [n][leg_output_width] f32 or NULL. */
int ovn_heads_forward(ovn_handle* h, const float* d_bank, int64_t bank_size,
                      const int32_t* d_left_idx, const int32_t* d_right_idx, int32_t n_pairs,
                      float* d_overlap, int32_t* d_yaw, float* d_corr, void* stream);

/* 1 query vs N candidates (Infer.infer_multiple, infer.py:162-203): RIGHT = the query volume
 * d_query [360][128] for every pair, LEFT = d_bank[cand_idx[p]] (cand_idx NULL = 0..n-1). */
int ovn_heads_1vsN(ovn_handle* h, const float* d_bank, int64_t bank_size, const float* d_query,
                   const int32_t* d_cand_idx, int32_t n_cand,
                   float* d_overlap, int32_t* d_yaw, float* d_corr, void* stream);

/* Rows [row_lo, row_hi) of the ordered all-pairs matrix of a bank (Infer.infer_multiple_vs_multiple,
 * infer.py:205-238, with every (first, second) combination; testing.py:237-272): for each row i,
 * RIGHT = d_bank[i] and LEFT = d_bank[j] for every j < bank_size.  The delta head is not symmetric in
 * (LEFT, RIGHT), so all ordered pairs are computed.  d_overlap / d_yaw: [row_hi - row_lo][bank_size].
 * The loop over rows runs inside the library (no per-row host round trip through the caller). */
int ovn_heads_rows_vs_bank(ovn_handle* h, const float* d_bank, int64_t bank_size, int64_t row_lo, int64_t row_hi,
                           float* d_overlap, int32_t* d_yaw, void* stream);

/* ---- best matches of each row, reduced on the device (loop-closure evaluation, DESIGN.md section 7) -------
 * A row's records are ordered by overlap, descending, then by index, ascending; NaN ranks above every number
 * and -0 equals +0.  Each record carries the overlap and yaw stored at its index.  Slots beyond min(k, the row's
 * length) hold index = -1, overlap = -1, yaw = 0.  Outputs: d_top_overlap f32 / d_top_index i32 / d_top_yaw i32,
 * each [rows][k].  k must be in [1, 32].  Every argument is checked before anything is launched
 * (OVN_ERR_INVALID_ARG).  The kernel is profiled as "rows_topk".
 *
 * ovn_rows_topk: the best k records of each row of a caller's score matrix, e.g. ovn_heads_rows_vs_bank's output.
 * Row r is d_overlap / d_yaw [r * stride, r * stride + h_n[r]); h_n: host, [rows], each in [0, stride]. */
int ovn_rows_topk(ovn_handle* h, const float* d_overlap, const int32_t* d_yaw, int64_t rows, int64_t stride,
                  const int32_t* h_n /* [rows], host */, int32_t k, float* d_top_overlap, int32_t* d_top_index,
                  int32_t* d_top_yaw, void* stream);

/* ovn_heads_prefix_topk: for each row i in [row_lo, row_hi), ovn_heads_1vsN with query d_bank[i] (RIGHT) against
 * the candidates [0, h_n_cand[i - row_lo]) (LEFT), then the best k records of that row, index = candidate j.
 * The rows' scores go to a handle-owned scratch of at most 2^21 pairs (16 MiB, allocated by the first call); one
 * k_rows_topk launch reduces the rows the scratch holds whenever the next row does not fit, so only the [rows][k]
 * records leave the call.  h_n_cand: host, [row_hi - row_lo], each in [0, bank_size]. */
int ovn_heads_prefix_topk(ovn_handle* h, const float* d_bank, int64_t bank_size, int64_t row_lo, int64_t row_hi,
                          const int32_t* h_n_cand /* [row_hi - row_lo], host */, int32_t k, float* d_top_overlap,
                          int32_t* d_top_index, int32_t* d_top_yaw, void* stream);

/* ---- overlap-based Monte Carlo localization (overlapnet_b200/mcl.py, DESIGN.md sections 4 and 7) ---------------
 * A particle filter over planar poses (x, y, theta), float64, with float64 log-weights, on the device.  The map is K
 * keyframes and a raster [rows][cols] whose cell (r, c) covers x0 + c cell <= x < x0 + (c + 1) cell, likewise y from
 * y0, and holds the index of the keyframe nearest to its centre, or -1.  Random numbers: Philox4x32-10 keyed by the
 * seed, counter (particle, step, stream, block); stream 0 motion, 1 initialisation, 2 resampling.  Every reduction
 * runs in an order fixed by N: the same seed, map, observations and N give bit-identical particles and estimates.
 *   ovn_mcl_set_map: h_keyframes [K][3] (x, y, theta), h_raster [rows][cols] with entries in [-1, K); cell > 0 and
 *                    finite.  Synchronous; drops the particle set.
 *   ovn_mcl_init:    n particles, 1 <= n <= 2^24.  OVN_MCL_INIT_GLOBAL: keyframe floor(u K), uniform in the disk of
 *                    init_radius around it, theta uniform; h_pose / h_sigma ignored.  OVN_MCL_INIT_POSE: Gaussian
 *                    around h_pose [3] with standard deviations h_sigma [3] (each >= 0).  Log-weights -log n.
 *   ovn_mcl_predict: moves every particle by the odometry h_odom [3] (dx, dy, dtheta in the previous query frame) with
 *                    noise h_sigma [3] (>= 0), looks up its keyframe and writes the touched keyframes, ascending, to
 *                    d_touched [K]; *h_n_touched = their number.  Synchronous.
 *   ovn_mcl_update:  the heads' overlap d_overlap [n] and yaw d_yaw [n] (180 - argmax) of LEFT = keyframe d_touched[j],
 *                    RIGHT = the query; n must be the last predict's count (the pointers may be NULL when it is 0).
 *                    Adds each particle's log-likelihood, normalises, and resamples systematically when the ESS falls
 *                    below rho N.  sigma_overlap, sigma_yaw > 0 (radians), rho in [0, 1].  Synchronous: *h_est.
 *                    An observed overlap that is not finite, or an update after which no particle has a finite
 *                    log-weight, is OVN_ERR_INVALID_ARG (the message names which): the particle set and *h_est are
 *                    unchanged, the predict still awaits its update and only its stages are held.
 *   ovn_mcl_copy_particles: d_out [4][N] float64 x, y, theta, log-weight of the current set, asynchronous.
 *   ovn_mcl_copy_stage: d_out = a stage of the last step, asynchronous: MOTION [3][N] f64 (x, y, theta after the last
 *                    predict), LOOKUP [N] i32 (the keyframe of each particle after it, -1 outside), LOGLIK [N] f64,
 *                    WEIGHTS [N] f64 (the normalised weights), PREFIX [N] f64 (their inclusive prefix sum) and
 *                    ANCESTORS [N] i32 of the last update, the last two only when it resampled; SCALARS [8] f64 of the
 *                    last update: the max m of the updated log-weights, S = sum exp(lw - m), the ESS, x, y, theta,
 *                    the resampling decision (1 or 0) and the resampling offset u0.
 *   ovn_mcl_philox:  d_out [n][4] = the Philox4x32-10 words of the counters d_ctr [n][4] under the seed (tests).
 * Invalid arguments, a call before ovn_mcl_set_map / ovn_mcl_init, an update without a predict and a stage the handle
 * does not hold are OVN_ERR_INVALID_ARG with nothing launched; the handle stays usable. */
typedef enum ovn_mcl_init_mode {
  OVN_MCL_INIT_GLOBAL = 0,
  OVN_MCL_INIT_POSE = 1
} ovn_mcl_init_mode;
typedef enum ovn_mcl_stage {
  OVN_MCL_STAGE_MOTION = 0,
  OVN_MCL_STAGE_LOOKUP = 1,
  OVN_MCL_STAGE_LOGLIK = 2,
  OVN_MCL_STAGE_WEIGHTS = 3,
  OVN_MCL_STAGE_PREFIX = 4,
  OVN_MCL_STAGE_ANCESTORS = 5,
  OVN_MCL_STAGE_SCALARS = 6
} ovn_mcl_stage;
typedef struct ovn_mcl_estimate {
  double x, y, theta;             /* weighted means; theta = atan2(sum w sin, sum w cos) */
  double ess;                     /* 1 / sum w^2 before resampling */
  int32_t n_touched;              /* keyframes the heads scored */
  int32_t resampled;              /* 1 when the update resampled */
  int64_t step;                   /* predicts since ovn_mcl_init */
} ovn_mcl_estimate;
int ovn_mcl_set_map(ovn_handle* h, const double* h_keyframes, int32_t n_keyframes, const int32_t* h_raster,
                    int32_t rows, int32_t cols, double x0, double y0, double cell);
int ovn_mcl_init(ovn_handle* h, int32_t mode, int32_t n, uint64_t seed, const double* h_pose, const double* h_sigma,
                 double init_radius, void* stream);
int ovn_mcl_predict(ovn_handle* h, const double* h_odom, const double* h_sigma, int32_t* d_touched,
                    int32_t* h_n_touched, void* stream);
int ovn_mcl_update(ovn_handle* h, const float* d_overlap, const int32_t* d_yaw, int32_t n, double sigma_overlap,
                   double sigma_yaw, double rho, ovn_mcl_estimate* h_est, void* stream);
int ovn_mcl_copy_particles(ovn_handle* h, double* d_out, void* stream);
int ovn_mcl_copy_stage(ovn_handle* h, int32_t stage, void* d_out, void* stream);
int ovn_mcl_philox(ovn_handle* h, uint64_t seed, const uint32_t* d_ctr, int32_t n, uint32_t* d_out, void* stream);

/* ---- point-to-plane ICP of loop-closure pairs on range images (overlapnet_b200/registration.py, DESIGN.md
 * sections 4 and 7).  Reference: none (the paper's ICP verification of loop candidates, seeded by the yaw head).
 * Pair i registers the source scan d_src[i] (RIGHT) to the target scan d_dst[i] (LEFT): it estimates the row-major
 * float64 pose T = T_LEFT^-1 T_RIGHT that takes the source's vertices into the target's frame, starting from the
 * first three rows of d_init[i] ([np][16]).  The images are what ovn_project_batch / ovn_normals_batch write at the
 * handle's geometry: d_vertex [n_scans][H][W][4] (w = 1 where valid) and d_normal [n_scans][H][W][3] ((-1, -1, -1)
 * where absent).  Per iteration k, with d_k = max(d_end, d_start gamma^k): a valid source pixel is moved by T in
 * float64 and binned by the ground-truth generator's float64 range_projection (dropped outside (0, max_range)); it
 * is an inlier when that target pixel is valid, ||p - q|| <= d_k and n_t . (R n_s) >= cos_normal.  The 29 float64
 * sums of H = sum J^T J (upper triangle, row by row), g = sum J e, the inliers and sum e^2, with e = n_t . (p - q)
 * and J = [p x n_t, n_t], give the update H delta = -g (Cholesky) applied on the left, T <- [R(omega) | v] T.  A pair
 * ends CONVERGED once d_k = d_end and ||omega|| < eps_rot and ||v|| < eps_trans, DEGENERATE at a pivot <= 1e-12
 * trace(H), TOO_FEW_INLIERS below min_inliers, else MAX_ITERATIONS.  One CTA runs every iteration of a pair and sums
 * in a fixed order, so a pair's result has the same bits in any batch, position, call or handle.
 *   d_out [np]: the pose, rms = sqrt(sum e^2 / inliers), inliers and the sums of the last iteration run, the valid
 *               source pixels, the iterations run and the status.
 *   d_assoc [np][H][W] (optional, NULL to skip): the inlier target pixel by * W + bx of each source pixel, or -1, in
 *               the last iteration run.  d_system [np][29] (optional): that iteration's sums before its solve.  With
 *               iterations = 1 both are exactly one step from d_init.
 * NULL pointers, np < 0, n_scans < 1 with np > 0, iterations outside [1, 200], min_inliers < 0, a parameter that is
 * not finite, d_end <= 0, d_end > d_start, gamma outside (0, 1], cos_normal outside [0, 1], eps_* < 0 and a d_init
 * value that is not finite (read back synchronously) are OVN_ERR_INVALID_ARG with nothing launched; np = 0 is a
 * no-op.  An index outside [0, n_scans) raises the device flag (ovn_check), and only its pair is poisoned: NaN pose
 * and rms, status OVN_ICP_BAD_INDEX, d_assoc -1, d_system NaN. */
#define OVN_ICP_SYSTEM_SIZE 29
#define OVN_ICP_MAX_ITERATIONS_LIMIT 200
typedef enum ovn_icp_status {
  OVN_ICP_CONVERGED = 0,
  OVN_ICP_MAX_ITERATIONS = 1,
  OVN_ICP_DEGENERATE = 2,
  OVN_ICP_TOO_FEW_INLIERS = 3,
  OVN_ICP_BAD_INDEX = 4
} ovn_icp_status;
typedef struct ovn_icp_params {
  double d_start, d_end, gamma;   /* association distance schedule, metres: d_k = max(d_end, d_start gamma^k) */
  double cos_normal;              /* the least cosine between the target normal and the moved source normal */
  double eps_rot, eps_trans;      /* convergence: the update's rotation (rad) and translation (m) */
  int32_t iterations;             /* the most iterations, 1 .. 200 */
  int32_t min_inliers;
} ovn_icp_params;
typedef struct ovn_icp_result {
  double pose[16];                /* row-major T_LEFT^-1 T_RIGHT */
  double rms;                     /* of the last iteration's inlier residuals, metres */
  int32_t inliers;                /* of the last iteration */
  int32_t valid;                  /* valid source pixels (vertex and normal) */
  int32_t iterations;             /* iterations run */
  int32_t status;                 /* ovn_icp_status */
} ovn_icp_result;
/* defaults: 2 m -> 0.3 m, gamma 0.8, cos 30 deg, 1e-6 rad, 1e-5 m, 30 iterations, 100 inliers (not tuned on KITTI) */
void ovn_icp_default_params(ovn_icp_params* p);
int ovn_icp_pairs(ovn_handle* h, const float* d_vertex, const float* d_normal, int32_t n_scans, const int32_t* d_src,
                  const int32_t* d_dst, const double* d_init, int32_t np, const ovn_icp_params* params,
                  ovn_icp_result* d_out, int32_t* d_assoc, double* d_system, void* stream);

/* ---- robust pose-graph optimization of a batch of graphs (overlapnet_b200/pose_graph.py, DESIGN.md sections 4 and
 * 7, "Pose-graph optimization").  Reference: none; the model is DESIGN section 7's.
 * Graph g has the nodes [node_offset[g], node_offset[g + 1]) (n >= 2 of them) and the edges [edge_offset[g],
 * edge_offset[g + 1]); edge node indices are local to the graph.  Its first n - 1 edges are the odometry chain
 * (k, k + 1) in order; every later edge is a loop edge (a, b), a != b.  A node is a row-major float64 4x4 pose; node
 * 0 is fixed.  Edge k measures Z_k ~ T_a^-1 T_b with the weights w_k ((omega, v) order, > 0): its residual is
 * e = (Log(R_E), t_E) of E = Z^-1 T_a^-1 T_b, chi2 = e^T diag(w) e, and the cost is F = 1/2 sum rho(chi2) with
 * rho(x) = x on the chain and the Geman-McClure rho(x) = phi x / (phi + x) on loops (phi = +inf: rho(x) = x).
 * Levenberg-Marquardt on (H + lambda diag(H)) delta = -g over nodes 1 .. n-1, solved by conjugate gradients
 * preconditioned with the exact block Cholesky factor of the damped block-diagonal plus the chain's off-diagonal
 * blocks; each node moves as T <- [R(omega) | v] T.  One CTA runs every iteration of one graph and sums in a fixed
 * order, so a graph's outputs have the same bits in any batch, position, call or handle.
 * All buffers are host memory; the call copies in, runs one k_pgo_graphs launch on `stream` and copies out
 * synchronously; the launch is profiled as "pgo_graphs".  Outputs:
 *   out_poses [N][16]      the poses at the last accepted state
 *   out_result [n_graphs]  status, iterations (every LM trial), accepted trials, CG iterations, F at the input and
 *                          at the end, the final lambda and max |g| over nodes 1 .. n-1 at the end
 *   out_chi2, out_scale [E]  chi2 and s = phi / (phi + chi2) of each edge at the end (s = 1 on the chain)
 *   out_gradient [N][6]    (optional, NULL to skip) g of every node at the end, node 0 included
 *   out_trace [n_graphs][max_iterations] (optional) each trial's F, lambda, accepted flag and CG iterations;
 *                          slots past the graph's last trial hold NaN, NaN, -1, -1
 * With max_iterations = 0 the call only evaluates F, chi2, s and g at the input.
 * Refused with OVN_ERR_INVALID_ARG and nothing launched or written: NULL required pointers, n_graphs outside
 * [1, OVN_PGO_MAX_GRAPHS], offsets not starting at 0 or not increasing, a graph with n < 2, more than
 * OVN_PGO_MAX_NODES nodes or OVN_PGO_MAX_EDGES edges or fewer than n - 1 edges, a chain edge other than (k, k + 1),
 * a node index out of range or a == b, a pose or measurement that is not finite or whose bottom row is not
 * 0 0 0 1, a weight that is not finite or <= 0, and parameters out of their ranges (phi > 0, may be +inf;
 * 0 < lambda_min <= lambda0 <= lambda_max, finite; tolerances finite and >= 0; max_iterations in
 * [0, OVN_PGO_MAX_ITERATIONS_LIMIT]; max_cg_iterations in [1, OVN_PGO_MAX_CG_ITERATIONS_LIMIT]). */
#define OVN_PGO_MAX_GRAPHS 65535
#define OVN_PGO_MAX_NODES (1 << 20)
#define OVN_PGO_MAX_EDGES (1 << 22)
#define OVN_PGO_MAX_ITERATIONS_LIMIT 1000
#define OVN_PGO_MAX_CG_ITERATIONS_LIMIT 10000
typedef enum ovn_pgo_status {
  OVN_PGO_CONVERGED = 0,
  OVN_PGO_MAX_ITERATIONS = 1,
  OVN_PGO_STALLED = 2,          /* lambda > lambda_max */
  OVN_PGO_FAILED = 3            /* a non-positive preconditioner pivot or p^T (H + lambda D) p <= 0 */
} ovn_pgo_status;
typedef struct ovn_pgo_params {
  double phi;                     /* Geman-McClure scale of the loop edges; +inf: plain least squares */
  double lambda0, lambda_min, lambda_max;   /* LM damping, relative to diag(H) */
  double rel_cost_tol;            /* converged: an accepted step lowers F by at most rel_cost_tol F */
  double step_tol;                /* converged: max |delta| <= step_tol */
  double cg_tol;                  /* CG stops at ||r|| <= cg_tol ||g|| */
  int32_t max_iterations;         /* LM trials, 0 .. 1000 */
  int32_t max_cg_iterations;      /* per trial, 1 .. 10000 */
} ovn_pgo_params;
typedef struct ovn_pgo_result {
  double initial_cost, final_cost, lambda, max_gradient;
  int32_t status, iterations, accepted, cg_iterations;
} ovn_pgo_result;
typedef struct ovn_pgo_trial {
  double cost, lambda;            /* the trial's F and the lambda it was solved with */
  int32_t accepted, cg_iterations;
} ovn_pgo_trial;
/* defaults: phi 25, lambda 1e-6 in [1e-12, 1e12], rel_cost_tol 1e-10, step_tol 1e-10, cg_tol 1e-12, 50 iterations,
 * 2000 CG iterations (none tuned on KITTI) */
void ovn_pgo_default_params(ovn_pgo_params* p);
int ovn_pgo_optimize_host(ovn_handle* h, int32_t n_graphs, const int64_t* node_offset, const int64_t* edge_offset,
                          const double* poses, const int32_t* edge_nodes, const double* edge_pose,
                          const double* edge_weight, const ovn_pgo_params* params, double* out_poses,
                          ovn_pgo_result* out_result, double* out_chi2, double* out_scale, double* out_gradient,
                          ovn_pgo_trial* out_trace, void* stream);
/* ovn_pgo_copy_workspace: h_out = one array of graph `graph` of the last successful ovn_pgo_optimize_host call,
 * synchronously, as the kernel left it (DESIGN.md section 2, "Pose-graph stages").  n and E are the graph's nodes and
 * edges; every array is float64, per node or per edge, in the graph's local order:
 *   T, Tt [n][16]      the poses of the last accepted state and the last trial's poses
 *   M [E][36], q [E][6]  each edge's rho' A^T W A and rho' A^T W e at T
 *   Hd [n][36], gn [n][6]  each node's diagonal block and gradient at T
 *   Ld, Ls, Lk [n][36]  the preconditioner's Cholesky blocks of the last factor: Ld of nodes 1 .. n-1; Ls (the block
 *                      below node j) of the segment nodes that are not the last node n - 1; Lk (the spike to the left
 *                      separator, or of separator q >= 2 the block to separator q - 1) of the nodes of segments 1 .. Q
 *                      and of separators 2 .. Q
 *   x, r, z, p, Ap [n][6]  the last trial's CG vectors, y [n][6] its last forward substitution, nodes 1 .. n-1
 * Positions not listed (node 0 of Ld / Ls / Lk and of the vectors, Ls of the separators and of node n - 1, Lk of
 * segment 0 and of the first separator) are never written and hold data of earlier calls; so does every array but
 * T, M, q, Hd and gn after a call with max_iterations = 0 or whose trials all had g = 0.  After a trial is accepted
 * M, q, Hd and gn are those of the new T, while the factor and the vectors stay those of the trial.
 * Refused with OVN_ERR_INVALID_ARG: no successful call since the handle was created or since the last call that
 * returned an error, `graph` or `array` out of range, or h_out NULL. */
typedef enum ovn_pgo_array {
  OVN_PGO_T = 0, OVN_PGO_TT = 1, OVN_PGO_M = 2, OVN_PGO_Q = 3, OVN_PGO_HD = 4, OVN_PGO_GN = 5, OVN_PGO_LD = 6,
  OVN_PGO_LS = 7, OVN_PGO_LK = 8, OVN_PGO_X = 9, OVN_PGO_R = 10, OVN_PGO_Z = 11, OVN_PGO_P = 12, OVN_PGO_AP = 13,
  OVN_PGO_Y = 14
} ovn_pgo_array;
int ovn_pgo_copy_workspace(ovn_handle* h, int32_t array, int32_t graph, double* h_out);

/* ---- resident bank (Infer keeps self.feature_volumes across calls, infer.py:113,184-193) ---------
 * The tensor-core heads consume fp16 / hi-lo split copies of the LEFT volumes.  Without this call
 * they are rebuilt from d_bank on every heads call; ovn_bank_prepare builds them once for rows
 * [first, first+count) of the bank that lives at d_bank (capacity = rows the bank may grow to), and
 * every later ovn_heads_forward / ovn_heads_1vsN whose d_bank is the same pointer reuses them.
 * Call it again for rows that were appended or overwritten.  No-op for precision fp32. */
int ovn_bank_prepare(ovn_handle* h, const float* d_bank, int64_t bank_capacity, int64_t first, int64_t count,
                     void* stream);
int ovn_bank_release(ovn_handle* h, const float* d_bank);

/* ---- training of the overlap head with a frozen leg (training.py; legsType 360OutputkLegsFixed,
 * generateNet.py:222-324) ------------------------------------------------------------------------
 * c_conv1..3 and overlap_output are trained, the leg is never touched.  fp32 arithmetic; every reduction
 * runs in a fixed order, so identical calls give bit-identical weights.  The gradient, Adagrad-accumulator
 * and activation buffers are allocated when a handle first trains (sized by max_batch_pairs); the gradients and
 * accumulators then cover every layer, leg included.
 * Losses (training.py:71-92,255-257): L = 5 L_ov + L_or,
 *   L_ov = mean_p sigmoid((|overlap_p - gt_overlap_p| + 0.25) * 24 - 12),
 *   L_or = mean_p mean_k weighted_cross_entropy_with_logits(t_pk, corr_pk, pos_weight = 360),
 *   t_pk = 1 iff k == gt_orientation_p and gt_overlap_p > min_overlap_for_angle
 *   (ImagePairOverlapOrientationSequence.py:118-121).  With a frozen leg L_or has no gradient. */
/* fp32 handles only (OVN_ERR_BAD_CONFIG otherwise); n_pairs <= max_batch_pairs (OVN_ERR_CAPACITY).
 * Forward of both heads + losses + backward of the overlap head for LEFT = bank[left], RIGHT = bank[right].
 * Synchronous: h_loss[3] = {total, overlap, orientation}.  Leaves the batch gradients in the handle.
 * An index outside the bank returns OVN_ERR_INVALID_ARG and leaves no usable gradients. */
int ovn_head_gradients(ovn_handle* h, const float* d_bank, int64_t bank_size,
                       const int32_t* d_left_idx, const int32_t* d_right_idx, int32_t n_pairs,
                       const float* d_gt_overlap, const int32_t* d_gt_orientation,
                       float min_overlap_for_angle, float* h_loss, void* stream);
/* Adagrad update of c_conv1..3 / overlap_output from the last valid gradients (Keras 2.1.5:
 * a += g^2; w -= lr g / (sqrt(a) + 1e-7), accumulators start at 0); refuses (INVALID_ARG) when there are
 * none.  ovn_finalize_weights resets the accumulators.  One launch. */
int ovn_head_adagrad_step(ovn_handle* h, float learning_rate, void* stream);
/* ---- training of the whole network (legsType 360OutputkLegs, generateNet.py:119-219) ----------
 * fp32 handles only (OVN_ERR_BAD_CONFIG otherwise); n_pairs <= max_batch_pairs and n_pairs <= 485 at
 * leg_output_width 360 (the launch grid of the heads' c_conv1), else OVN_ERR_CAPACITY.
 * Forward of leg + both heads for LEFT = images[left], RIGHT = images[right] (d_images: [n_images][H][W][C]),
 * the losses of training.py, and the backward of the whole network: the correlation head's loss now reaches
 * the leg.  Synchronous: h_loss[3].  d_fv_grad (may be NULL) receives dL/d(LEFT volume), dL/d(RIGHT volume)
 * as [2][n_pairs][Wf][128], before s_conv10's ReLU mask.  An index outside the image bank returns
 * OVN_ERR_INVALID_ARG and leaves no usable gradients.  The per-batch buffers are allocated on the first call. */
int ovn_net_gradients(ovn_handle* h, const float* d_images, int64_t n_images,
                      const int32_t* d_left_idx, const int32_t* d_right_idx, int32_t n_pairs,
                      const float* d_gt_overlap, const int32_t* d_gt_orientation,
                      float min_overlap_for_angle, float* h_loss, float* d_fv_grad, void* stream);
/* The feature volumes of the last valid ovn_net_gradients batch, as its leg forward computed them (at the handle's
 * training precision): d_out [2][n_pairs][Wf][128], LEFT then RIGHT, asynchronous on `stream`.  fp32 handles
 * (OVN_ERR_BAD_CONFIG otherwise); OVN_ERR_INVALID_ARG when there is no such batch. */
int ovn_copy_net_volumes(ovn_handle* h, float* d_out, void* stream);
/* Adagrad over every leg and head layer from the last ovn_net_gradients; INVALID_ARG otherwise (also after an
 * ovn_head_gradients call).  The head layers share their accumulators with ovn_head_adagrad_step.  One launch. */
int ovn_net_adagrad_step(ovn_handle* h, float learning_rate, void* stream);
/* ---- training precision -------------------------------------------------------------------------------
 * The arithmetic of every GEMM-shaped product inside ovn_head_gradients and ovn_net_gradients, forward and
 * backward, and of the |l - r| backward of ovn_net_gradients.  OVN_TRAIN_FP32 (the default): fp32 SIMT FMAs.
 * OVN_TRAIN_TF32X3: tensor cores (mma.sync TF32).  Each operand x is split into x_hi = tf32(x) and
 * x_lo = tf32(x - x_hi), both rounded to nearest with ties away from zero; a product is
 * a_lo b_hi + a_hi b_lo + a_hi b_hi, accumulated in fp32; a_lo b_lo (at most 2^-22 |a b|) is dropped.  The
 * gradients stay fp32-grade (DESIGN.md section 2 gives the measured deviations) and two identical calls still
 * give bit-identical results.  Only those two gradient calls are affected: the correlation backward, the losses,
 * the Dense and ReLU backward, the split-K sums and every Adagrad step stay fp32, and so does every other entry
 * point (ovn_leg_forward, ovn_heads_forward, ...).  ovn_copy_gradients and ovn_adagrad_step_sum work on whatever
 * gradients the last gradient call left.  Allowed between any two calls.  OVN_ERR_BAD_CONFIG on a handle whose
 * precision is not OVN_PREC_FP32; OVN_ERR_INVALID_ARG for a value not in ovn_train_precision. */
typedef enum ovn_train_precision {
  OVN_TRAIN_FP32 = 0,
  OVN_TRAIN_TF32X3 = 1
} ovn_train_precision;
int ovn_set_train_precision(ovn_handle* h, int32_t train_precision);
/* ---- data-parallel training (overlapnet_b200/training.py, DESIGN.md section 6) --------------------------
 * Each rank computes the gradients of its share of a batch with ovn_head_gradients / ovn_net_gradients, copies
 * them into one flat float32 vector, the ranks exchange those vectors, and every rank applies the same
 * weighted sum to its weights.  The flat layout: c_conv1..3 and overlap_output, then (whole_network != 0) every
 * leg layer input to output; each layer [K + 1][N], its kernel in Keras layout, then its bias.
 *   ovn_train_gradient_size: *n = the number of floats of that vector (665 025 for the heads at the default
 *                    geometry; 1 769 137 for the whole network at C = 4 with s_conv3a).
 *   ovn_copy_gradients: d_out[n] = the gradients of the last valid ovn_head_gradients / ovn_net_gradients call,
 *                    asynchronous on `stream`.  fp32 handles (OVN_ERR_BAD_CONFIG otherwise); OVN_ERR_INVALID_ARG
 *                    when there are none, or when whole_network asks for leg layers after ovn_head_gradients.
 *   ovn_adagrad_step_sum: per element, in part order, g = w0 p0 + w1 p1 + ... (d_parts [n_parts][n], h_weights
 *                    [n_parts] on the host; each product and sum rounded to float32, no FMA contraction; parts
 *                    with weight 0 are skipped), then the update of ovn_head_adagrad_step (whole_network = 0) or
 *                    ovn_net_adagrad_step with g, rounded as those calls round it: a = fma(g, g, a);
 *                    w -= (lr g) / (sqrt(a) + 1e-7).  One part of weight 1 reproduces those calls bit for bit.
 *                    It does not need the handle's own gradients; fp32 handles and finalised weights only.
 *                    n_parts < 1 or a NULL pointer: OVN_ERR_INVALID_ARG; n_parts > 64: OVN_ERR_CAPACITY.  One
 *                    launch. */
int ovn_train_gradient_size(ovn_handle* h, int32_t whole_network, int64_t* n);
int ovn_copy_gradients(ovn_handle* h, int32_t whole_network, float* d_out, void* stream);
int ovn_adagrad_step_sum(ovn_handle* h, int32_t whole_network, const float* d_parts, int32_t n_parts,
                         const float* h_weights, float learning_rate, void* stream);
/* ---- gradients per chunk of a batch (gradient_chunks in overlapnet_b200/training.py, DESIGN.md section 6) -------
 * One call over the pairs [0, n_pairs) of a range, cut into n_chunks contiguous chunks: chunk c is the pairs
 * [h_chunk_offsets[c], h_chunk_offsets[c + 1]) (host array of n_chunks + 1).  d_parts [n_chunks][n] (n =
 * ovn_train_gradient_size(h, 0) for the heads call, (h, 1) for the whole-network call) and h_loss [n_chunks][3]:
 * part c and h_loss[c] are bit for bit what ovn_head_gradients / ovn_net_gradients on the pairs of chunk c alone
 * leave in h_loss and, through ovn_copy_gradients, in d_out -- at either training precision.  An empty chunk gives a
 * zero part and zero losses.  The stages that compute each pair on its own (the leg and heads forward, every input
 * gradient, the ReLU masks) run once over the range; the losses and every weight gradient run per chunk.
 * Synchronous, like the one-chunk calls.  The call leaves no gradients and no batch in the handle:
 * ovn_copy_gradients, ovn_copy_net_volumes, ovn_get_gradients, ovn_head_adagrad_step and ovn_net_adagrad_step
 * return OVN_ERR_INVALID_ARG until the next ovn_head_gradients / ovn_net_gradients; ovn_adagrad_step_sum takes
 * the parts.  Errors: those of the one-chunk calls for the whole range (n_pairs <= 485 at leg_output_width 360 for
 * the whole network), plus n_chunks < 1, a NULL h_chunk_offsets or d_parts, or offsets that do not run
 * non-decreasing from 0 to n_pairs (OVN_ERR_INVALID_ARG), and n_chunks > 64 (OVN_ERR_CAPACITY). */
int ovn_head_gradients_chunks(ovn_handle* h, const float* d_bank, int64_t bank_size,
                              const int32_t* d_left_idx, const int32_t* d_right_idx, int32_t n_pairs,
                              const int32_t* h_chunk_offsets, int32_t n_chunks,
                              const float* d_gt_overlap, const int32_t* d_gt_orientation,
                              float min_overlap_for_angle, float* d_parts, float* h_loss, void* stream);
int ovn_net_gradients_chunks(ovn_handle* h, const float* d_images, int64_t n_images,
                             const int32_t* d_left_idx, const int32_t* d_right_idx, int32_t n_pairs,
                             const int32_t* h_chunk_offsets, int32_t n_chunks,
                             const float* d_gt_overlap, const int32_t* d_gt_orientation,
                             float min_overlap_for_angle, float* d_parts, float* h_loss, void* stream);
/* ---- the training state, for checkpoints that resume a run (overlapnet_b200/training.py, DESIGN.md section 6) --
 * The Adagrad accumulators as one flat float32 vector in the layout of ovn_copy_gradients:
 * ovn_train_gradient_size(h, whole_network) floats, the heads' prefix (whole_network = 0) or every layer.
 *   ovn_copy_train_state: d_out[n] = the accumulators, asynchronous on `stream`.  A handle that never trained
 *                    returns zeros (what its first Adagrad step starts from).
 *   ovn_set_train_state: the accumulators = d_in[n], asynchronous on `stream`; allocates the training state when
 *                    the handle has none.  whole_network = 0 writes the heads' prefix only and leaves the leg's
 *                    accumulators as they are.  The values are not checked: a negative or non-finite one makes the
 *                    next Adagrad steps non-finite.
 * ovn_finalize_weights resets the accumulators to zero, so a resumed run sets its weights first (ovn_set_weights,
 * ovn_finalize_weights), then its state.  fp32 handles (OVN_ERR_BAD_CONFIG otherwise); OVN_ERR_INVALID_ARG for a
 * NULL pointer or when the weights are not finalised. */
int ovn_copy_train_state(ovn_handle* h, int32_t whole_network, float* d_out, void* stream);
int ovn_set_train_state(ovn_handle* h, int32_t whole_network, const float* d_in, void* stream);
/* ---- yaw augmentation of training images (DESIGN.md section 7) ------------------------------------
 * The reference's rotate_training_data rolls the RIGHT image by randint(0, width) columns but leaves its yaw
 * label where it was, and rolls the normal channels without rotating the vectors
 * (ImagePairOverlapOrientationSequence.py:76-80, 114-121, 209-212).  This is the geometric version: rolling a
 * range image by s columns is the image of the cloud rotated about z by theta = -2 pi s / W (utils.py:86-90),
 * so the normals are rotated by theta too and the caller moves the label by -s Wf / W bins.
 * d_out[i][y][x][c] = d_images[d_rows[i]][y][(x - d_shift[i]) mod W][c] for i < n; the normal channels get
 * (nx, ny) -> (cos nx - sin ny, sin nx + cos ny) with d_rot[i] = (cos theta, sin theta), rounded like NumPy's
 * float32 (no FMA); a normal pixel equal to the fill (-1, -1, -1) and every other channel are copied.
 * d_shift NULL = every shift 0, d_rot NULL = normals not rotated.  A row outside [0, n_images) is clamped and
 * reported as OVN_ERR_INVALID_ARG by the next ovn_check.  Both precisions. */
int ovn_gather_images(ovn_handle* h, const float* d_images, int64_t n_images, const int32_t* d_rows,
                      const int32_t* d_shift, const float* d_rot /* [n][2] */, int32_t n,
                      float* d_out /* [n][H][W][C] */, void* stream);
/* ---- a training image bank in host memory (overlapnet_b200/image_bank.py, DESIGN.md section 6) ---------------
 *   ovn_train_workspace_bytes: *bytes = the device memory the training buffers of this handle take once it has
 *                    trained n_pairs-pair batches: the heads' buffers, gradients and accumulators, and with
 *                    whole_network the leg activations of 2 n_pairs images and their backward buffers; the split-K
 *                    partials counted once.  Allocates nothing.
 *   ovn_host_register / ovn_host_unregister: page-lock (cudaHostRegister, portable) / release `bytes` of host
 *                    memory the caller owns, so that copies from it are asynchronous.  OVN_ERR_CUDA with the
 *                    runtime's message when the pin fails.
 *   ovn_stage_rows:  for i < n, one cudaMemcpyAsync on `stream` of row h_rows[i] (row_bytes bytes) of the host
 *                    block h_src [n_src_rows][row_bytes] to d_dst + i row_bytes.  h_rows is read on the host before
 *                    any copy is issued; a row outside [0, n_src_rows) is OVN_ERR_INVALID_ARG and nothing is
 *                    copied.  h_src must be page-locked for the copies to be asynchronous.  Both precisions. */
int ovn_train_workspace_bytes(ovn_handle* h, int32_t whole_network, int32_t n_pairs, int64_t* bytes);
int ovn_host_register(ovn_handle* h, void* h_ptr, int64_t bytes);
int ovn_host_unregister(ovn_handle* h, void* h_ptr);
int ovn_stage_rows(ovn_handle* h, const void* h_src, int64_t n_src_rows, int64_t row_bytes, const int64_t* h_rows,
                   int32_t n, void* d_dst, void* stream);
/* ---- a training image bank sharded over the GPUs of a node (overlapnet_b200/image_bank.py, DESIGN.md section 6) --
 * Each rank holds a contiguous block of the bank's rows in a shard of its own device memory; a step's rows are
 * gathered into a device slot straight from the owners' memory (over NVLink, or within one device).
 *   ovn_shard_create: allocates a shard of `bytes` > 0 bytes, owned by the handle: one cudaMalloc of exactly that
 *                    size, so that *d_ptr is the allocation's base.  Writes its CUDA IPC handle (cudaIpcGetMemHandle,
 *                    64 bytes) to h_ipc.  OVN_ERR_CUDA with the runtime's message when either call fails.
 *   ovn_shard_open:  maps another process's shard from its 64-byte IPC handle (cudaIpcOpenMemHandle, peer access
 *                    enabled lazily); the mapping is owned by the handle.  A handle that cannot be opened (a device
 *                    without peer access, a zeroed or stale handle, a shard of this same process) is OVN_ERR_CUDA
 *                    with the runtime's message; nothing is mapped and the handle stays usable.
 *   ovn_shard_close: synchronises the device, then unmaps a shard ovn_shard_open mapped or frees one
 *                    ovn_shard_create allocated.  Any other pointer is OVN_ERR_INVALID_ARG.  The caller makes sure
 *                    no other process still reads an own shard (a barrier after every rank closed its mappings).
 *                    ovn_destroy closes the remaining mappings before it frees the remaining own shards.
 *   ovn_gather_rows: for i < n, d_dst + i row_bytes = row h_rows[i] (row_bytes bytes) of the bank of which shard s
 *                    (a device pointer: own or mapped) holds rows [h_first[s], h_first[s + 1]).  One launch of
 *                    k_gather_rows on `stream` per 1024 rows, 16-byte loads and stores; the source of every row
 *                    travels in the launch's parameters, so the host arrays may be reused once the call returns.
 *                    Checked on the host before anything is issued: n < 0, n_shards < 1, h_first not starting at
 *                    0 or decreasing, row_bytes not a positive multiple of 16, a NULL or not 16-byte aligned shard
 *                    pointer or d_dst, a row outside [0, h_first[n_shards]) are OVN_ERR_INVALID_ARG and nothing is
 *                    copied.  Both precisions; profiled as "gather_rows". */
int ovn_shard_create(ovn_handle* h, int64_t bytes, void** d_ptr, void* h_ipc /* 64 bytes */);
int ovn_shard_open(ovn_handle* h, const void* h_ipc /* 64 bytes */, void** d_ptr);
int ovn_shard_close(ovn_handle* h, void* d_ptr);
int ovn_gather_rows(ovn_handle* h, const void* const* h_shards, const int64_t* h_first /* [n_shards + 1] */,
                    int32_t n_shards, int64_t row_bytes, const int64_t* h_rows, int32_t n, void* d_dst, void* stream);
/* Current weights / last gradients of a layer, Keras layout, host buffers (same shapes as ovn_set_weights).
 * Both synchronise the device.  ovn_get_gradients returns the head layers after ovn_head_gradients and every
 * layer after ovn_net_gradients. */
int ovn_get_weights(ovn_handle* h, const char* layer_name, float* h_kernel, float* h_bias);
int ovn_get_gradients(ovn_handle* h, const char* layer_name, float* h_kernel, float* h_bias);

/* ---- deferred device errors ------------------------------------------------------------------
 * The device-pointer entry points never synchronise, so three classes of error can only be detected on
 * the device: an index outside [0, bank_size) (or, for a resident bank, a row that was never
 * prepared), a volume value the fp16 operands of the tensor-core heads cannot hold (NaN, inf, or more
 * than 65504 away from the feature centre; raised by every heads call that reads such a volume -- a
 * resident bank row keeps its mark from ovn_bank_prepare until it is prepared again) or, in the
 * tensor-core leg (ovn_leg_forward and the *_host entry points at precision f16_tc), an input pixel that
 * is NaN or inf or an activation of any layer but the last above 65504, which the hi / lo fp16 planes
 * between the layers cannot hold (the feature volumes of that call are not valid: without the flag the
 * next layer's ReLU would turn the NaN into ordinary zeros), and a bounded
 * pipeline-barrier wait of a tensor-core kernel that timed out (GPU time-slicing, debuggers).  Each raises
 * a flag on the device; the kernels that write overlap / yaw
 * then POISON their outputs (overlap = NaN, yaw = INT32_MIN) so garbage never looks valid, indices are
 * clamped so no out-of-bounds read happens, and the flag is turned into a status by the next entry point
 * that synchronises anyway: ovn_check (synchronises `stream`), the *_host entry points and
 * ovn_profile_read.  OVN_ERR_INVALID_ARG for index and value errors, OVN_ERR_CUDA for time-outs; the flag is
 * cleared when it is reported. */
int ovn_check(ovn_handle* h, void* stream);

/* ---- device-side signalling between the GPUs of a sharded bank (overlapnet_b200/search.py, transport 'symm') --
 * The query volume and the result table of a sharded 1-vs-N search live in symmetric (peer-mapped) memory:
 * kernels read / write them directly over NVLink, and these two calls replace the collectives.  A flag is an
 * int32 slot in that memory holding the number of the last finished step.
 *   ovn_peer_signal: ONE launch stores `value` (release, system scope -- after everything queued on `stream`
 *                    before it) to each of the n flag addresses (host array of peer-mapped device addresses).
 *   ovn_peer_wait:   ONE launch spins (acquire, system scope, bounded) until d_flags[i] >= value for every
 *                    i < n except i == skip.  A time-out raises the handle's deferred error (ovn_check). */
int ovn_peer_signal(ovn_handle* h, const uint64_t* h_flag_ptrs, int32_t n, int32_t value, void* stream);
int ovn_peer_wait(ovn_handle* h, const int32_t* d_flags, int32_t n, int32_t skip, int32_t value, void* stream);

/* ---- feature centre of the tensor-core delta head ------------------------------------------------
 * DeltaLayer only sees |l - r| (generateNet.py:59), which is invariant to a common per-channel offset:
 * the fp16 operand copies of the volumes are stored as fp16(x - mu[c]), which shrinks their rounding
 * error (3x on leg outputs in a float64 emulation of the rounding, tools/precision_study.py).  mu is calibrated automatically
 * on the first volume the handle sees (first ovn_bank_prepare row, else the first RIGHT volume) and
 * then frozen until ovn_finalize_weights; ovn_set_feature_center(h, mu[128]) fixes it explicitly
 * (NULL = back to automatic; not allowed while a bank is resident).  No effect for precision fp32. */
int ovn_set_feature_center(ovn_handle* h, const float* h_mu);
int ovn_get_feature_center(ovn_handle* h, float* h_mu /* [128] */, int32_t* is_set);
/* The same offset trick is applied to the two intermediate images (o1, x3: c_conv2 and c_conv3 are
 * linear, the mean's image is folded into the layer's bias with exact fp32 weights).  All three centres are
 * derived from ONE feature volume V0 with fixed summation orders: mu = channel means of V0, the o1 / x3
 * centres = channel means over the canonical pair (V0, V0 rolled by half a turn).  V0 is the first volume
 * the handle sees, or the one given here: ovn_calibrate(h, d_volume [360][128]) makes the calibration
 * explicit, so that handles on different GPUs (a sharded bank) produce bit-identical results. */
int ovn_calibrate(ovn_handle* h, const float* d_volume, void* stream);

/* ---- intermediate stages of the tensor-core heads (tests and diagnostics) -------------------------
 * The stages are what the last chunk of the last heads call (ovn_heads_forward, ovn_heads_1vsN,
 * ovn_heads_rows_vs_bank, ovn_query_cloud_vs_bank_host; a chunk is at most max_batch_pairs pairs) left in
 * the handle.  ovn_heads_stage_pairs: *n_pairs = the pairs of that chunk, 0 when there are none (before the
 * first heads call, after a calibration -- ovn_calibrate or the one a first ovn_bank_prepare runs -- which
 * overwrites o1 and x3, and after a heads call that returned an error).  ovn_copy_heads_stage: d_out (float32,
 * device) = pairs [first, first + count) of one stage, exactly count x the per-pair size below (CENTRES:
 * first and count are ignored); pairs outside [0, n_pairs) are OVN_ERR_INVALID_ARG.  A plain copy and
 * conversion of the stored values, asynchronous on `stream`:
 *   OVN_STAGE_O1      [count][Wf=360][24][64] (i, jb, o): the fp16 c_conv1 output k_delta_conv1_wgmma stored,
 *                     without the c_conv1 bias and minus the o1 centre
 *   OVN_STAGE_X3      [count][24][24][128] (ib, jb, c): the fp16 ReLU(c_conv2) minus the x3 centre
 *   OVN_STAGE_DENSE   [count][24][24][2] (ib, jb, half): the Dense(1) partial sum of each c_conv3 output pixel
 *                     over output channels [128 half, 128 half + 128); exactly 0 where ib or jb >= 22
 *   OVN_STAGE_CENTRES [64 + 128 + 128 + 256]: o1 centre, x3 centre, c_conv2 bias with both centres folded in
 *                     (b2eff), c_conv3 bias with the x3 centre folded in (b3eff)
 * Both return OVN_ERR_BAD_CONFIG on a precision fp32 handle.  The heads calls do no extra work for this. */
typedef enum ovn_heads_stage {
  OVN_STAGE_O1 = 0,
  OVN_STAGE_X3 = 1,
  OVN_STAGE_DENSE = 2,
  OVN_STAGE_CENTRES = 3
} ovn_heads_stage;
int ovn_heads_stage_pairs(ovn_handle* h, int64_t* n_pairs);
int ovn_copy_heads_stage(ovn_handle* h, int32_t stage, int64_t first, int64_t count, float* d_out, void* stream);

/* ---- one layer of the tensor-core leg (tests and diagnostics) --------------------------------------
 * Runs ovn_leg_forward's own launch sequence on n_scans <= max_batch_scans scans (the same kernels, grids and
 * K slices as a leg call of that many scans) and stops after leg layer `layer` (0 = s_conv1 ... the last layer
 * but one; the last layer's float32 volume is ovn_leg_forward).  d_hi, d_lo (float32, device)
 * [n_scans][h_out][w_out][cout] of that layer = the fp16 halves of its activation as stored for the next layer,
 * hi = fp16(v), lo = fp16(v - hi), converted exactly.  OVN_ERR_BAD_CONFIG on a precision fp32 handle,
 * OVN_ERR_WEIGHTS before ovn_finalize_weights, OVN_ERR_INVALID_ARG for a layer or n_scans out of range. */
int ovn_leg_stage(ovn_handle* h, const float* d_input, int32_t n_scans, int32_t layer, float* d_hi, float* d_lo,
                  void* stream);

/* ---- stages of a training step (tests and diagnostics; oracle/train_stages.py, DESIGN.md section 4) ---------
 * The buffers of the last ovn_head_gradients / ovn_net_gradients call (chunked forms included) of n_pairs pairs,
 * read back as float32.  Wf = leg_output_width, s = conv1size, nb = Wf / s, nit = ceil(Wf / 64); "images order" is
 * the order of the gathered images: chunk after chunk, the chunk's LEFT images then its RIGHT images (one chunk:
 * LEFT 0..n-1, RIGHT 0..n-1).
 * Stop stages: values the step overwrites later in place.  ovn_set_train_stop(h, stage, layer) makes the next
 * gradient call stop right after that value is complete (stage = -1: no stop); the stop is consumed by that call
 * whatever it returns, and a stop its flow never reaches (a whole-network stage in ovn_head_gradients) lets the
 * call run to the end.  A call that stopped writes no losses and leaves no gradients and no batch:
 * ovn_get_gradients, ovn_copy_gradients, ovn_copy_net_volumes, ovn_head_adagrad_step, ovn_net_adagrad_step and
 * ovn_adagrad_step_sum return OVN_ERR_INVALID_ARG until a call runs to the end; the parts of a stopped _chunks call
 * are incomplete.  The next whole call computes exactly what it computes on a fresh handle.
 *   OVN_TRAIN_STAGE_O1        [n][Wf][nb][64] (i, jb, o) c_conv1 output with its bias
 *   OVN_TRAIN_STAGE_X4        [n][o3_h][o3_w][256] ReLU(c_conv3), the Dense input
 *   OVN_TRAIN_STAGE_DFV_CORR  [2][n][Wf][128] (LEFT, RIGHT) dL/d(volumes) of the correlation head (k_corr_backward)
 *   OVN_TRAIN_STAGE_LEG_DY    layer l: [2n][h_out][w_out][cout] in images order, dL/d(pre-activation of leg layer l)
 *                             (the top layer's is the |l - r| and correlation parts summed, masked by the volumes)
 * Stages read after a call that ran to the end:
 *   OVN_TRAIN_STAGE_X3        [n][o2_h][o2_w][128] ReLU(c_conv2)
 *   OVN_TRAIN_STAGE_OVERLAP   [n] yhat;  OVN_TRAIN_STAGE_CORR [n][Wf] orientation logits
 *   OVN_TRAIN_STAGE_DZ        [n] dL/d(Dense logit), each chunk's own 1 / n
 *   OVN_TRAIN_STAGE_DPRE3     [n][o3_h][o3_w][256] dL/d(pre-activation of c_conv3)
 *   OVN_TRAIN_STAGE_DX3       [n][o2_h][o2_w][128] dL/d(pre-activation of c_conv2)
 *   OVN_TRAIN_STAGE_DO1       [n][o2_h][nb][s][64] (ho, jb, dh, o) dL/d(c_conv1 output) at row i = s ho + dh
 *   OVN_TRAIN_STAGE_DCORR     [n][Wf] dL/d(orientation logits)                       (whole network only, so on)
 *   OVN_TRAIN_STAGE_PART_L    [n][nb][Wf][128] k_delta_dgrad partials of dL/dLEFT, one per jb
 *   OVN_TRAIN_STAGE_PART_R    [n][nit][Wf][128] partials of dL/dRIGHT, one per 64-row tile of i
 *   OVN_TRAIN_STAGE_IMAGES    [2n][H][W][C] the gathered images, images order
 *   OVN_TRAIN_STAGE_ACT       layer l: [2n][h_out][w_out][cout] leg layer l's output, images order
 * ovn_train_stage_size: *n = the floats of the stage; ovn_copy_train_stage: d_out[*n] = the stage, asynchronous on
 * `stream`.  Both OVN_ERR_INVALID_ARG for a stage the handle does not hold: no successful gradient call, a
 * whole-network stage after ovn_head_gradients, a stop stage other than the one the call stopped at, or any other
 * stage after a stopped call.  layer is the leg layer (0 = s_conv1) for LEG_DY and ACT, 0 for every other stage.
 * fp32 handles (OVN_ERR_BAD_CONFIG otherwise).  The gradient calls issue the same launches with or without a
 * readback; a stop only ends the call early. */
typedef enum ovn_train_stage {
  OVN_TRAIN_STAGE_O1 = 0,
  OVN_TRAIN_STAGE_X4 = 1,
  OVN_TRAIN_STAGE_DFV_CORR = 2,
  OVN_TRAIN_STAGE_LEG_DY = 3,
  OVN_TRAIN_STAGE_X3 = 4,
  OVN_TRAIN_STAGE_OVERLAP = 5,
  OVN_TRAIN_STAGE_CORR = 6,
  OVN_TRAIN_STAGE_DZ = 7,
  OVN_TRAIN_STAGE_DPRE3 = 8,
  OVN_TRAIN_STAGE_DX3 = 9,
  OVN_TRAIN_STAGE_DO1 = 10,
  OVN_TRAIN_STAGE_DCORR = 11,
  OVN_TRAIN_STAGE_PART_L = 12,
  OVN_TRAIN_STAGE_PART_R = 13,
  OVN_TRAIN_STAGE_IMAGES = 14,
  OVN_TRAIN_STAGE_ACT = 15
} ovn_train_stage;
int ovn_set_train_stop(ovn_handle* h, int32_t stage, int32_t layer);
int ovn_train_stage_size(ovn_handle* h, int32_t stage, int32_t layer, int64_t* n);
int ovn_copy_train_stage(ovn_handle* h, int32_t stage, int32_t layer, float* d_out, void* stream);

/* ---- host-buffer convenience entry points (what a non-CUDA caller binds; bench.py e2e) ------ */
/* Raw clouds on the host -> feature volumes on the host.  OVN_ERR_BAD_CONFIG on a handle with
 * probability channels. */
int ovn_encode_clouds_host(ovn_handle* h, const float* h_points, const int64_t* h_offsets,
                           int32_t n_scans, float* h_fv);
/* One raw query cloud on the host vs a device-resident bank: preprocess + leg + heads.
 * h_overlap [n_cand], h_yaw [n_cand]; h_query_fv [360][128] may be NULL.  OVN_ERR_BAD_CONFIG on a
 * handle with probability channels. */
int ovn_query_cloud_vs_bank_host(ovn_handle* h, const float* h_points, int64_t n_points,
                                 const float* d_bank, int64_t bank_size,
                                 const int32_t* h_cand_idx, int32_t n_cand,
                                 float* h_overlap, int32_t* h_yaw, float* h_query_fv);
/* The same two with per-point class probabilities, through ovn_preprocess_cues_batch: the semantic
 * cue as gen_semantic_data.py:33-46 makes it from the clouds and their .label files.  h_probs:
 * [n_points][n_prob_channels] float32 host rows, one per point of h_points, in the same order;
 * required iff the handle has probability channels (else NULL; OVN_ERR_INVALID_ARG).  The rows are
 * staged next to the cloud (80 B per point at 20 classes); the query keeps its one host
 * synchronisation. */
int ovn_encode_clouds_probs_host(ovn_handle* h, const float* h_points, const int64_t* h_offsets,
                                 int32_t n_scans, const float* h_probs, float* h_fv);
int ovn_query_cloud_probs_vs_bank_host(ovn_handle* h, const float* h_points, int64_t n_points,
                                       const float* h_probs, const float* d_bank, int64_t bank_size,
                                       const int32_t* h_cand_idx, int32_t n_cand,
                                       float* h_overlap, int32_t* h_yaw, float* h_query_fv);

#ifdef __cplusplus
}
#endif
#endif /* OVN_B200_H_ */
