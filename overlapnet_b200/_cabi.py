"""ctypes binding of include/ovn_b200.h.  The product path has NO CPU fallback: if the shared
library is missing or a call fails, an exception is raised."""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, 'libovn_b200.so')

OVN_ABI_VERSION = 1
PREC_FP32 = 0
PREC_F16_TC = 1

# every symbol include/ovn_b200.h declares (tests/test_cabi.py checks the .so exports them all)
SYMBOLS = [
    'ovn_default_config', 'ovn_create', 'ovn_destroy', 'ovn_last_error', 'ovn_status_string',
    'ovn_abi_version', 'ovn_input_channels', 'ovn_feature_width', 'ovn_feature_channels',
    'ovn_launch_count', 'ovn_profile_enable', 'ovn_profile_read', 'ovn_set_weights', 'ovn_finalize_weights', 'ovn_project_batch',
    'ovn_normals_batch', 'ovn_semantic_batch', 'ovn_gt_range_batch', 'ovn_gt_overlap_count', 'ovn_gt_scan_radius',
    'ovn_gt_pairs_count', 'ovn_preprocess_batch', 'ovn_preprocess_cues_batch', 'ovn_render_batch',
    'ovn_render_preprocess_batch', 'ovn_surfel_default_params', 'ovn_surfels_batch', 'ovn_render_surfels_batch',
    'ovn_render_surfels_preprocess_batch',
    'ovn_pack_input',
    'ovn_leg_forward', 'ovn_heads_forward', 'ovn_heads_1vsN', 'ovn_bank_prepare', 'ovn_bank_release', 'ovn_encode_clouds_host',
    'ovn_query_cloud_vs_bank_host', 'ovn_check', 'ovn_set_feature_center', 'ovn_get_feature_center',
    'ovn_heads_rows_vs_bank', 'ovn_calibrate', 'ovn_peer_signal', 'ovn_peer_wait',
    'ovn_head_gradients', 'ovn_head_adagrad_step', 'ovn_get_weights', 'ovn_get_gradients',
    'ovn_net_gradients', 'ovn_net_adagrad_step', 'ovn_gather_images',
    'ovn_train_gradient_size', 'ovn_copy_gradients', 'ovn_adagrad_step_sum', 'ovn_set_train_precision',
    'ovn_copy_net_volumes', 'ovn_copy_train_state', 'ovn_set_train_state',
    'ovn_train_workspace_bytes', 'ovn_host_register', 'ovn_host_unregister', 'ovn_stage_rows',
    'ovn_head_gradients_chunks', 'ovn_net_gradients_chunks', 'ovn_copy_heads_stage',
    'ovn_heads_stage_pairs', 'ovn_leg_stage', 'ovn_encode_clouds_probs_host', 'ovn_query_cloud_probs_vs_bank_host',
    'ovn_shard_create', 'ovn_shard_open', 'ovn_shard_close', 'ovn_gather_rows',
    'ovn_set_train_stop', 'ovn_train_stage_size', 'ovn_copy_train_stage',
    'ovn_rows_topk', 'ovn_heads_prefix_topk',
    'ovn_mcl_set_map', 'ovn_mcl_init', 'ovn_mcl_predict', 'ovn_mcl_update', 'ovn_mcl_copy_particles',
    'ovn_mcl_copy_stage', 'ovn_mcl_philox', 'ovn_icp_default_params', 'ovn_icp_pairs',
    'ovn_pgo_default_params', 'ovn_pgo_optimize_host', 'ovn_pgo_copy_workspace',
]
TOPK_MAX = 32     # ovn_rows_topk / ovn_heads_prefix_topk: k in [1, TOPK_MAX]
MCL_INIT_MODES = {'global': 0, 'pose': 1}     # ovn_mcl_init_mode
MCL_STAGES = {'motion': 0, 'lookup': 1, 'loglik': 2, 'weights': 3, 'prefix': 4, 'ancestors': 5,
              'scalars': 6}                                                                      # ovn_mcl_stage
MCL_MAX_PARTICLES = 1 << 24
ICP_SYSTEM_SIZE = 29      # ovn_icp_pairs: d_system [np][ICP_SYSTEM_SIZE]
ICP_STATUS = {'converged': 0, 'max_iterations': 1, 'degenerate': 2, 'too_few_inliers': 3, 'bad_index': 4}     # ovn_icp_status
PGO_STATUS = {'converged': 0, 'max_iterations': 1, 'stalled': 2, 'failed': 3}     # ovn_pgo_status
PGO_MAX_GRAPHS = 65535
PGO_MAX_NODES = 1 << 20
PGO_MAX_EDGES = 1 << 22
PGO_MAX_ITERATIONS = 1000
PGO_MAX_CG_ITERATIONS = 10000
# ovn_pgo_array: name -> (value, doubles per node or edge, per edge)
PGO_ARRAYS = {'T': (0, 16, False), 'Tt': (1, 16, False), 'M': (2, 36, True), 'q': (3, 6, True), 'Hd': (4, 36, False),
              'gn': (5, 6, False), 'Ld': (6, 36, False), 'Ls': (7, 36, False), 'Lk': (8, 36, False),
              'x': (9, 6, False), 'r': (10, 6, False), 'z': (11, 6, False), 'p': (12, 6, False), 'Ap': (13, 6, False),
              'y': (14, 6, False)}
IPC_HANDLE_BYTES = 64     # ovn_shard_create / ovn_shard_open
HEADS_STAGES = {'o1': 0, 'x3': 1, 'dense': 2, 'centres': 3}     # ovn_heads_stage
TRAIN_PRECISIONS = {'fp32': 0, 'tf32x3': 1}     # ovn_train_precision
TRAIN_STAGES = {'o1': 0, 'x4': 1, 'dfv_corr': 2, 'leg_dy': 3, 'x3': 4, 'overlap': 5, 'corr': 6, 'dz': 7,
                'dpre3': 8, 'dx3': 9, 'do1': 10, 'dcorr': 11, 'part_l': 12, 'part_r': 13, 'images': 14,
                'act': 15}      # ovn_train_stage
TRAIN_STOPS = ('o1', 'x4', 'dfv_corr', 'leg_dy')


class OvnConfig(C.Structure):
  _fields_ = [
      ('abi_version', C.c_int32),
      ('proj_H', C.c_int32), ('proj_W', C.c_int32),
      ('fov_up_deg', C.c_float), ('fov_down_deg', C.c_float), ('max_range', C.c_float),
      ('use_depth', C.c_int32), ('use_normals', C.c_int32), ('n_prob_channels', C.c_int32),
      ('use_intensity', C.c_int32),
      ('strides_layer1', C.c_int32 * 2),
      ('additional_unsymmetric_layer3a', C.c_int32),
      ('leg_output_width', C.c_int32),
      ('conv1size', C.c_int32),
      ('precision', C.c_int32),
      ('max_batch_scans', C.c_int32), ('max_batch_pairs', C.c_int32),
  ]


class McEstimate(C.Structure):
  """ovn_mcl_estimate"""
  _fields_ = [('x', C.c_double), ('y', C.c_double), ('theta', C.c_double), ('ess', C.c_double),
              ('n_touched', C.c_int32), ('resampled', C.c_int32), ('step', C.c_int64)]


class IcpParams(C.Structure):
  """ovn_icp_params"""
  _fields_ = [('d_start', C.c_double), ('d_end', C.c_double), ('gamma', C.c_double), ('cos_normal', C.c_double),
              ('eps_rot', C.c_double), ('eps_trans', C.c_double), ('iterations', C.c_int32), ('min_inliers', C.c_int32)]


class PgoParams(C.Structure):
  """ovn_pgo_params"""
  _fields_ = [('phi', C.c_double), ('lambda0', C.c_double), ('lambda_min', C.c_double), ('lambda_max', C.c_double),
              ('rel_cost_tol', C.c_double), ('step_tol', C.c_double), ('cg_tol', C.c_double),
              ('max_iterations', C.c_int32), ('max_cg_iterations', C.c_int32)]


class PgoResult(C.Structure):
  """ovn_pgo_result"""
  _fields_ = [('initial_cost', C.c_double), ('final_cost', C.c_double), ('lambda_', C.c_double),
              ('max_gradient', C.c_double), ('status', C.c_int32), ('iterations', C.c_int32), ('accepted', C.c_int32),
              ('cg_iterations', C.c_int32)]


class PgoTrial(C.Structure):
  """ovn_pgo_trial"""
  _fields_ = [('cost', C.c_double), ('lambda_', C.c_double), ('accepted', C.c_int32), ('cg_iterations', C.c_int32)]


class SurfelParams(C.Structure):
  """ovn_surfel_params"""
  _fields_ = [('kappa', C.c_double), ('c_min', C.c_double), ('max_splat', C.c_int32)]


SURFEL_MAX_SPLAT = 32     # ovn_surfel_params.max_splat in [0, SURFEL_MAX_SPLAT]
SURFEL_FLOATS = 8         # ovn_surfels_batch: d_surfels [n][H][W][SURFEL_FLOATS]
ICP_RESULT_BYTES = 152    # sizeof(ovn_icp_result): pose double[16], rms double, inliers, valid, iterations, status int32


class OvnError(Exception):
  """Raised for any non-zero ovn_status (plain Exception subclass, like the reference's errors)."""


_lib = None


def lib():
  """Load libovn_b200.so (built in-tree by overlapnet_b200.build).  Fails loudly when absent."""
  global _lib
  if _lib is not None:
    return _lib
  if not os.path.exists(LIB_PATH):
    raise OvnError('libovn_b200.so is not built: run `python -m overlapnet_b200.build` '
                   '(there is no CPU fallback for the CUDA path)')
  L = C.CDLL(LIB_PATH)
  vp, i32, i64, f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_float
  u64, f64 = C.c_uint64, C.c_double
  L.ovn_default_config.argtypes = [C.POINTER(OvnConfig)]
  L.ovn_default_config.restype = None
  L.ovn_create.argtypes = [C.POINTER(OvnConfig), C.POINTER(vp)]
  L.ovn_destroy.argtypes = [vp]
  L.ovn_last_error.argtypes = [vp]
  L.ovn_last_error.restype = C.c_char_p
  L.ovn_status_string.argtypes = [C.c_int]
  L.ovn_status_string.restype = C.c_char_p
  L.ovn_abi_version.restype = C.c_int
  for f in ('ovn_input_channels', 'ovn_feature_width', 'ovn_feature_channels'):
    getattr(L, f).argtypes = [vp]
  L.ovn_launch_count.argtypes = [vp]
  L.ovn_launch_count.restype = i64
  L.ovn_profile_enable.argtypes = [vp, C.c_int]
  L.ovn_profile_read.argtypes = [vp, C.c_char_p, C.POINTER(C.c_double), C.POINTER(i64)]
  L.ovn_set_weights.argtypes = [vp, C.c_char_p, vp, C.POINTER(i64), i32, vp, i64]
  L.ovn_finalize_weights.argtypes = [vp]
  L.ovn_project_batch.argtypes = [vp, vp, vp, i32, i64, f32, vp, vp, vp, vp, vp]
  L.ovn_normals_batch.argtypes = [vp, vp, vp, i32, vp, vp]
  L.ovn_gt_range_batch.argtypes = [vp, vp, vp, i32, i64, vp, vp, f32, vp, vp]
  L.ovn_gt_overlap_count.argtypes = [vp, vp, vp, i32, vp, vp]
  L.ovn_gt_scan_radius.argtypes = [vp, vp, vp, i32, vp, vp]
  L.ovn_gt_pairs_count.argtypes = [vp, vp, vp, i32, vp, vp, vp, vp, i32, f32, i32, i32, vp, i64, vp, vp]
  L.ovn_semantic_batch.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp]
  L.ovn_preprocess_batch.argtypes = [vp, vp, vp, i32, i64, vp, vp, vp]
  L.ovn_preprocess_cues_batch.argtypes = [vp, vp, vp, i32, i64, vp, vp, vp]
  L.ovn_render_batch.argtypes = [vp, vp, vp, i32, i32, vp, vp, vp, f32, vp, vp, vp, vp, vp]
  L.ovn_render_preprocess_batch.argtypes = [vp, vp, vp, i32, i32, vp, vp, vp, vp, vp]
  L.ovn_surfel_default_params.argtypes = [C.POINTER(SurfelParams)]
  L.ovn_surfel_default_params.restype = None
  L.ovn_surfels_batch.argtypes = [vp, vp, vp, i32, i64, C.POINTER(SurfelParams), vp, vp]
  L.ovn_render_surfels_batch.argtypes = [vp, vp, i32, vp, i32, vp, vp, vp, C.POINTER(SurfelParams), f32, vp, vp, vp,
                                         vp, vp]
  L.ovn_render_surfels_preprocess_batch.argtypes = [vp, vp, i32, vp, i32, vp, vp, vp, C.POINTER(SurfelParams), vp, vp]
  L.ovn_pack_input.argtypes = [vp, vp, vp, vp, vp, i32, vp, vp]
  L.ovn_leg_forward.argtypes = [vp, vp, i32, vp, vp]
  L.ovn_heads_forward.argtypes = [vp, vp, i64, vp, vp, i32, vp, vp, vp, vp]
  L.ovn_heads_1vsN.argtypes = [vp, vp, i64, vp, vp, i32, vp, vp, vp, vp]
  L.ovn_bank_prepare.argtypes = [vp, vp, i64, i64, i64, vp]
  L.ovn_heads_rows_vs_bank.argtypes = [vp, vp, i64, i64, i64, vp, vp, vp]
  L.ovn_rows_topk.argtypes = [vp, vp, vp, i64, i64, vp, i32, vp, vp, vp, vp]
  L.ovn_heads_prefix_topk.argtypes = [vp, vp, i64, i64, i64, vp, i32, vp, vp, vp, vp]
  L.ovn_mcl_set_map.argtypes = [vp, vp, i32, vp, i32, i32, f64, f64, f64]
  L.ovn_mcl_init.argtypes = [vp, i32, i32, u64, vp, vp, f64, vp]
  L.ovn_mcl_predict.argtypes = [vp, vp, vp, vp, C.POINTER(i32), vp]
  L.ovn_mcl_update.argtypes = [vp, vp, vp, i32, f64, f64, f64, C.POINTER(McEstimate), vp]
  L.ovn_mcl_copy_particles.argtypes = [vp, vp, vp]
  L.ovn_mcl_copy_stage.argtypes = [vp, i32, vp, vp]
  L.ovn_mcl_philox.argtypes = [vp, u64, vp, i32, vp, vp]
  L.ovn_icp_default_params.argtypes = [C.POINTER(IcpParams)]
  L.ovn_icp_default_params.restype = None
  L.ovn_icp_pairs.argtypes = [vp, vp, vp, i32, vp, vp, vp, i32, C.POINTER(IcpParams), vp, vp, vp, vp]
  L.ovn_pgo_default_params.argtypes = [C.POINTER(PgoParams)]
  L.ovn_pgo_default_params.restype = None
  L.ovn_pgo_optimize_host.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, C.POINTER(PgoParams), vp, vp, vp, vp, vp, vp,
                                      vp]
  L.ovn_pgo_copy_workspace.argtypes = [vp, i32, i32, vp]
  L.ovn_bank_release.argtypes = [vp, vp]
  L.ovn_check.argtypes = [vp, vp]
  L.ovn_set_feature_center.argtypes = [vp, vp]
  L.ovn_get_feature_center.argtypes = [vp, vp, C.POINTER(i32)]
  L.ovn_calibrate.argtypes = [vp, vp, vp]
  L.ovn_copy_heads_stage.argtypes = [vp, i32, i64, i64, vp, vp]
  L.ovn_heads_stage_pairs.argtypes = [vp, C.POINTER(i64)]
  L.ovn_leg_stage.argtypes = [vp, vp, i32, i32, vp, vp, vp]
  L.ovn_set_train_stop.argtypes = [vp, i32, i32]
  L.ovn_train_stage_size.argtypes = [vp, i32, i32, C.POINTER(i64)]
  L.ovn_copy_train_stage.argtypes = [vp, i32, i32, vp, vp]
  L.ovn_peer_signal.argtypes = [vp, vp, i32, i32, vp]
  L.ovn_peer_wait.argtypes = [vp, vp, i32, i32, i32, vp]
  L.ovn_head_gradients.argtypes = [vp, vp, i64, vp, vp, i32, vp, vp, f32, vp, vp]
  L.ovn_head_adagrad_step.argtypes = [vp, f32, vp]
  L.ovn_net_gradients.argtypes = [vp, vp, i64, vp, vp, i32, vp, vp, f32, vp, vp, vp]
  L.ovn_net_adagrad_step.argtypes = [vp, f32, vp]
  L.ovn_gather_images.argtypes = [vp, vp, i64, vp, vp, vp, i32, vp, vp]
  L.ovn_train_gradient_size.argtypes = [vp, i32, C.POINTER(i64)]
  L.ovn_copy_gradients.argtypes = [vp, i32, vp, vp]
  L.ovn_adagrad_step_sum.argtypes = [vp, i32, vp, i32, vp, f32, vp]
  L.ovn_set_train_precision.argtypes = [vp, i32]
  L.ovn_copy_net_volumes.argtypes = [vp, vp, vp]
  L.ovn_copy_train_state.argtypes = [vp, i32, vp, vp]
  L.ovn_set_train_state.argtypes = [vp, i32, vp, vp]
  L.ovn_train_workspace_bytes.argtypes = [vp, i32, i32, C.POINTER(i64)]
  L.ovn_host_register.argtypes = [vp, vp, i64]
  L.ovn_host_unregister.argtypes = [vp, vp]
  L.ovn_stage_rows.argtypes = [vp, vp, i64, i64, vp, i32, vp, vp]
  L.ovn_shard_create.argtypes = [vp, i64, C.POINTER(vp), vp]
  L.ovn_shard_open.argtypes = [vp, vp, C.POINTER(vp)]
  L.ovn_shard_close.argtypes = [vp, vp]
  L.ovn_gather_rows.argtypes = [vp, vp, vp, i32, i64, vp, i32, vp, vp]
  L.ovn_head_gradients_chunks.argtypes = [vp, vp, i64, vp, vp, i32, vp, i32, vp, vp, f32, vp, vp, vp]
  L.ovn_net_gradients_chunks.argtypes = [vp, vp, i64, vp, vp, i32, vp, i32, vp, vp, f32, vp, vp, vp]
  L.ovn_get_weights.argtypes = [vp, C.c_char_p, vp, vp]
  L.ovn_get_gradients.argtypes = [vp, C.c_char_p, vp, vp]
  L.ovn_encode_clouds_host.argtypes = [vp, vp, vp, i32, vp]
  L.ovn_query_cloud_vs_bank_host.argtypes = [vp, vp, i64, vp, i64, vp, i32, vp, vp, vp]
  L.ovn_encode_clouds_probs_host.argtypes = [vp, vp, vp, i32, vp, vp]
  L.ovn_query_cloud_probs_vs_bank_host.argtypes = [vp, vp, i64, vp, vp, i64, vp, i32, vp, vp, vp]
  _lib = L
  return L


def check(handle, status, what=''):
  if status != 0:
    L = lib()
    msg = L.ovn_last_error(handle).decode(errors='replace') if L.ovn_last_error(handle) else ''
    raise OvnError('%s failed: %s (%s)' % (what or 'ovn call', L.ovn_status_string(status).decode(), msg))
