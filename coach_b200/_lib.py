"""ctypes binding of libcoach_b200.so (include/coach_b200.h).

There is NO fallback: if the CUDA library is missing or does not load, every compute path of ``coach_b200``
raises.  Build it with ``python -m coach_b200.build`` (or ``__graft_entry__.build()``).
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# CB200_LIB_PATH: load another build of the same library (an A/B build, for instance)
LIB_PATH = os.environ.get("CB200_LIB_PATH") or os.path.join(_HERE, "lib", "libcoach_b200.so")

c_void_p = ctypes.c_void_p
c_i64 = ctypes.c_int64
c_int = ctypes.c_int
c_double = ctypes.c_double
c_float = ctypes.c_float

CB200_MAX_COLUMNS = 8


class GemmDesc(ctypes.Structure):
    """struct cb200_gemm_desc"""
    _fields_ = [("a_src", c_void_p), ("a_lut", c_void_p), ("a_rowoff", c_void_p), ("a_coloff", c_void_p),
                ("a_rowinfo", c_void_p), ("a_colinfo", c_void_p), ("a_oh", ctypes.c_int32), ("a_ow", ctypes.c_int32),
                ("a_rows", ctypes.c_int32), ("a_cols", ctypes.c_int32), ("a_transposed", ctypes.c_int32),
                ("b", c_void_p), ("ldb", ctypes.c_int32), ("n", ctypes.c_int32),
                ("c", c_void_p), ("ldc", ctypes.c_int32), ("bias", c_void_p), ("act", ctypes.c_int32),
                ("mask_y", c_void_p), ("mask_act", ctypes.c_int32), ("c_rowmap", c_void_p),
                ("accumulate", ctypes.c_int32), ("workspace", c_void_p), ("splits", ctypes.c_int32),
                ("a_vec4", ctypes.c_int32), ("a_ones_col", ctypes.c_int32), ("a_u8_div", c_float),
                ("b_planes", c_void_p), ("b_plane_stride", c_i64), ("b_prow_npix", ctypes.c_int32),
                ("b_prow_batch", ctypes.c_int32), ("c_planes", c_void_p), ("c_plane_stride", c_i64),
                ("c_plane_cols", ctypes.c_int32), ("c_prow_npix", ctypes.c_int32), ("c_prow_batch", ctypes.c_int32),
                ("a_lda", ctypes.c_int32)]


class TGemmDesc(ctypes.Structure):
    """struct cb200_tgemm_desc"""
    _fields_ = [("mode", ctypes.c_int32), ("batch", ctypes.c_int32), ("a_planes", c_void_p), ("a_plane_stride", c_i64),
                ("a_cols", ctypes.c_int32), ("b_planes", c_void_p), ("b_plane_stride", c_i64), ("n", ctypes.c_int32),
                ("list_ptr", c_void_p), ("list", c_void_p), ("max_list_len", ctypes.c_int32), ("a_pix", c_void_p),
                ("num_q", ctypes.c_int32), ("taps", ctypes.c_int32), ("c", c_void_p), ("ldc", ctypes.c_int32),
                ("bias", c_void_p), ("act", ctypes.c_int32), ("mask_y", c_void_p), ("mask_act", ctypes.c_int32),
                ("c_rowmap", c_void_p), ("workspace", c_void_p), ("splits", ctypes.c_int32), ("c_planes", c_void_p),
                ("c_plane_stride", c_i64), ("c_plane_cols", ctypes.c_int32), ("mask_planes", c_void_p),
                ("mask_plane_stride", c_i64), ("bias_row", ctypes.c_int32),
                ("a_num_planes", ctypes.c_int32),
                ("a_u8_div", c_float), ("a_rows", c_i64), ("b_rows", c_i64),
                ("b_interleaved", ctypes.c_int32), ("a_pix_host", c_void_p), ("tmap_key", ctypes.c_uint64),
                ("a_tma", ctypes.c_int32), ("a_tile_class", ctypes.c_uint8 * 64),
                ("tmap_storage", ctypes.c_uint8 * (4 * 128 + 64))]


class DqnHeadDesc(ctypes.Structure):
    """struct cb200_dqn_head_desc"""
    _fields_ = [("h_next", c_void_p), ("h_online", c_void_p), ("h_select", c_void_p), ("w_target", c_void_p),
                ("b_target", c_void_p), ("w_online", c_void_p), ("b_online", c_void_p), ("actions", c_void_p),
                ("rewards", c_void_p), ("game_overs", c_void_p), ("weights", c_void_p), ("discount", c_double),
                ("huber", ctypes.c_int32), ("batch", c_i64), ("features", ctypes.c_int32),
                ("n_actions", ctypes.c_int32), ("q_online", c_void_p), ("q_next", c_void_p), ("targets", c_void_p),
                ("td_err", c_void_p), ("dq", c_void_p), ("loss", c_void_p), ("dh", c_void_p), ("dh_planes", c_void_p),
                ("dh_plane_stride", c_i64), ("dw", c_void_p), ("db", c_void_p), ("workspace", c_void_p),
                ("target_rule", ctypes.c_int32), ("h_target_s", c_void_p), ("mc_returns", c_void_p),
                ("pal_alpha", c_double), ("mc_mixing_rate", c_double), ("q_select", c_void_p),
                ("q_target_s", c_void_p)]


# cb200_dqn_head_desc.target_rule
TARGET_DQN, TARGET_MMC, TARGET_PAL, TARGET_PAL_PERSISTENT = 0, 1, 2, 3


class EnsembleHeadDesc(ctypes.Structure):
    """struct cb200_ensemble_head_desc"""
    _fields_ = [("h_next", c_void_p), ("h_online", c_void_p), ("h_select", c_void_p), ("w_target", c_void_p),
                ("b_target", c_void_p), ("w_online", c_void_p), ("b_online", c_void_p), ("actions", c_void_p),
                ("rewards", c_void_p), ("game_overs", c_void_p), ("masks", c_void_p), ("discount", c_double),
                ("huber", ctypes.c_int32), ("batch", c_i64), ("features", ctypes.c_int32), ("heads", ctypes.c_int32),
                ("n_actions", ctypes.c_int32), ("grad_rescale", c_float), ("q_online", c_void_p),
                ("q_next", c_void_p), ("q_select", c_void_p), ("targets", c_void_p), ("dq", c_void_p),
                ("losses", c_void_p), ("loss", c_void_p), ("dh", c_void_p), ("dh_planes", c_void_p),
                ("dh_plane_stride", c_i64), ("dw", c_void_p), ("db", c_void_p), ("workspace", c_void_p)]


class NafHeadDesc(ctypes.Structure):
    """struct cb200_naf_head_desc"""
    _fields_ = [("z_v", c_void_p), ("z_mu", c_void_p), ("l", c_void_p), ("scale", c_void_p), ("actions", c_void_p),
                ("targets", c_void_p), ("huber", ctypes.c_int32), ("batch", c_i64), ("n_actions", ctypes.c_int32),
                ("ld_mu", ctypes.c_int32), ("ld_l", ctypes.c_int32), ("ld_actions", ctypes.c_int32),
                ("mu", c_void_p), ("q", c_void_p), ("loss", c_void_p), ("d_zv", c_void_p), ("d_zmu", c_void_p),
                ("d_l", c_void_p), ("adv", c_void_p)]


class QrHeadDesc(ctypes.Structure):
    """struct cb200_qr_head_desc"""
    _fields_ = [("next", c_void_p), ("online", c_void_p), ("actions", c_void_p), ("rewards", c_void_p),
                ("game_overs", c_void_p), ("discount", c_double), ("kappa", c_float), ("batch", ctypes.c_int32),
                ("n_actions", ctypes.c_int32), ("n_atoms", ctypes.c_int32), ("dq", c_void_p), ("loss", c_void_p),
                ("targets", c_void_p), ("taus", c_void_p), ("target_actions", c_void_p), ("workspace", c_void_p)]


class NstepQHeadDesc(ctypes.Structure):
    """struct cb200_nstep_q_head_desc"""
    _fields_ = [("h_online", c_void_p), ("h_boot", c_void_p), ("w_target", c_void_p), ("b_target", c_void_p),
                ("w_online", c_void_p), ("b_online", c_void_p), ("actions", c_void_p), ("rewards", c_void_p),
                ("game_overs", c_void_p), ("seg_offsets", c_void_p), ("seg_lengths", c_void_p),
                ("segments", ctypes.c_int32), ("rows", c_i64), ("discount", c_double), ("horizon", ctypes.c_int32),
                ("huber", ctypes.c_int32), ("features", ctypes.c_int32), ("n_actions", ctypes.c_int32),
                ("q_online", c_void_p), ("dq", c_void_p), ("loss", c_void_p), ("targets", c_void_p),
                ("bootstrap", c_void_p), ("dh", c_void_p), ("dh_planes", c_void_p), ("dh_plane_stride", c_i64),
                ("dw", c_void_p), ("db", c_void_p), ("workspace", c_void_p)]


# cb200_nstep_q_head_desc.horizon
NSTEP_NONE, NSTEP_NSTEP, NSTEP_ONESTEP = 0, 1, 2


class ActorCriticHeadDesc(ctypes.Structure):
    """struct cb200_actor_critic_head_desc"""
    _fields_ = [("h", c_void_p), ("h_boot", c_void_p), ("w", c_void_p), ("b", c_void_p), ("actions", c_void_p),
                ("rewards", c_void_p), ("game_overs", c_void_p), ("seg_offsets", c_void_p), ("seg_lengths", c_void_p),
                ("segments", ctypes.c_int32), ("rows", c_i64), ("discount", c_double), ("gae_lambda", c_double),
                ("mode", ctypes.c_int32), ("huber", ctypes.c_int32), ("beta_entropy", c_float),
                ("v_weight", c_float), ("p_weight", c_float), ("features", ctypes.c_int32),
                ("n_actions", ctypes.c_int32), ("z", c_void_p), ("dz", c_void_p), ("loss", c_void_p),
                ("probs", c_void_p), ("targets", c_void_p), ("advantages", c_void_p), ("bootstrap", c_void_p),
                ("dh", c_void_p), ("dh_planes", c_void_p), ("dh_plane_stride", c_i64), ("dw", c_void_p),
                ("db", c_void_p), ("workspace", c_void_p)]


# cb200_actor_critic_head_desc.mode
AC_A_VALUE, AC_GAE, AC_GAE_VALUE = 0, 1, 2


class ActorCriticGaussianHeadDesc(ctypes.Structure):
    """struct cb200_actor_critic_gaussian_head_desc"""
    _fields_ = [("h", c_void_p), ("h_boot", c_void_p), ("w", c_void_p), ("b", c_void_p), ("actions", c_void_p),
                ("max_abs_range", c_void_p), ("rewards", c_void_p), ("game_overs", c_void_p),
                ("seg_offsets", c_void_p), ("seg_lengths", c_void_p), ("segments", ctypes.c_int32), ("rows", c_i64),
                ("discount", c_double), ("gae_lambda", c_double), ("mode", ctypes.c_int32),
                ("huber", ctypes.c_int32), ("beta_entropy", c_float), ("v_weight", c_float), ("p_weight", c_float),
                ("features", ctypes.c_int32), ("action_dim", ctypes.c_int32), ("z", c_void_p), ("dz", c_void_p),
                ("loss", c_void_p), ("means", c_void_p), ("stds", c_void_p), ("targets", c_void_p),
                ("advantages", c_void_p), ("bootstrap", c_void_p), ("dh", c_void_p), ("dh_planes", c_void_p),
                ("dh_plane_stride", c_i64), ("dw", c_void_p), ("db", c_void_p), ("workspace", c_void_p)]


def acg_workspace_floats(rows, segments, features, action_dim):
    """the floats cb200_actor_critic_gaussian_head's workspace takes"""
    N, chunks = 1 + 2 * action_dim, (rows + 63) // 64
    return rows * (N + 4) + segments + chunks * (features * N + N + 1)


class PolicyGradientHeadDesc(ctypes.Structure):
    """struct cb200_policy_gradient_head_desc"""
    _fields_ = [("h", c_void_p), ("w", c_void_p), ("b", c_void_p), ("targets", c_void_p), ("actions", c_void_p),
                ("cont_actions", c_void_p), ("max_abs_range", c_void_p), ("seg_offsets", c_void_p),
                ("seg_lengths", c_void_p), ("segments", ctypes.c_int32), ("rows", c_i64),
                ("continuous", ctypes.c_int32), ("features", ctypes.c_int32), ("n_outputs", ctypes.c_int32),
                ("beta_entropy", c_float), ("z", c_void_p), ("policy", c_void_p), ("dz", c_void_p),
                ("loss", c_void_p), ("dh", c_void_p), ("dh_planes", c_void_p), ("dh_plane_stride", c_i64),
                ("dw", c_void_p), ("db", c_void_p), ("workspace", c_void_p)]


# cb200_pg_targets rescalers (the values of PolicyGradientRescaler)
PG_TOTAL_RETURN, PG_FUTURE_RETURN, PG_NORMALIZED_BY_EPISODE, PG_NORMALIZED_BY_TIMESTEP = 0, 1, 2, 3


# cb200_ensemble_action_values modes
ENSEMBLE_SELECT, ENSEMBLE_UCB, ENSEMBLE_MEAN, ENSEMBLE_VOTE = 0, 1, 2, 3


class Column(ctypes.Structure):
    """struct cb200_column"""
    _fields_ = [("src", c_void_p), ("dst", c_void_p), ("row_bytes", c_i64)]


# name -> (restype, argtypes); every symbol of include/coach_b200.h (tests/test_cabi.py checks the two stay in sync)
PROTOTYPES = {
    "cb200_abi_version": (c_int, []),
    "cb200_last_error": (ctypes.c_char_p, []),
    "cb200_last_dispatch": (ctypes.c_char_p, []),
    "cb200_launch_count": (c_i64, []),
    "cb200_device_info": (c_int, [ctypes.POINTER(c_int)] * 3),
    "cb200_tune": (c_int, [ctypes.c_char_p, c_int]),
    "cb200_l2_persist": (c_int, [c_void_p, c_i64, c_void_p]),
    "cb200_per_init": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_void_p]),
    "cb200_per_update": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_void_p, c_void_p, c_void_p, c_i64,
                                 c_void_p, c_void_p, c_void_p]),
    "cb200_per_priorities_device": (c_int, [c_void_p, c_i64, c_double, c_double, c_void_p, c_void_p, c_void_p,
                                            c_void_p]),
    "cb200_host_priorities": (c_int, [c_void_p, c_i64, c_double, c_double, c_void_p, c_void_p]),
    "cb200_per_store": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_i64, c_double, c_double,
                                c_void_p]),
    "cb200_per_sample": (c_int, [c_void_p, c_void_p, c_i64, c_void_p, c_i64, c_i64, c_double, c_void_p, c_void_p,
                                 c_void_p, c_void_p]),
    "cb200_gather": (c_int, [ctypes.POINTER(Column), c_int, c_void_p, c_i64, c_void_p]),
    "cb200_per_sample_gather": (c_int, [c_void_p, c_void_p, c_i64, c_void_p, c_i64, c_i64, c_double, c_void_p,
                                        c_void_p, c_void_p, ctypes.POINTER(Column), c_int, c_void_p]),
    "cb200_per_sample_gather_s2d": (c_int, [c_void_p, c_void_p, c_i64, c_void_p, c_i64, c_i64, c_double, c_void_p,
                                            c_void_p, c_void_p, ctypes.POINTER(Column), c_int, ctypes.c_int32,
                                            ctypes.c_int32, ctypes.c_int32, ctypes.c_int32, ctypes.POINTER(Column),
                                            c_int, c_void_p, c_i64, c_void_p]),
    "cb200_gather_s2d": (c_int, [c_void_p, c_i64, ctypes.POINTER(Column), c_int, ctypes.c_int32, ctypes.c_int32,
                                 ctypes.c_int32, ctypes.c_int32, ctypes.POINTER(Column), c_int, c_void_p, c_i64,
                                 c_void_p]),
    "cb200_gather_stack": (c_int, [c_void_p, c_i64, c_void_p, ctypes.c_int32, c_void_p, c_i64, c_void_p, c_void_p]),
    "cb200_scatter_ring": (c_int, [ctypes.POINTER(Column), c_int, c_i64, c_i64, c_i64, c_void_p]),
    "cb200_scatter_ring_packed": (c_int, [ctypes.POINTER(Column), c_int, c_i64, c_i64, c_i64, c_i64, c_void_p]),
    "cb200_gemm": (c_int, [ctypes.POINTER(GemmDesc), c_void_p]),
    "cb200_colsum": (c_int, [c_void_p, c_i64, c_i64, c_void_p, c_void_p, c_void_p]),
    "cb200_permute_f32": (c_int, [c_void_p, c_void_p, c_i64, c_void_p, c_void_p, c_i64, c_int, c_void_p]),
    "cb200_gemm_tiled": (c_int, [c_void_p, c_void_p]),
    "cb200_u8_s2d_planes": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "cb200_transpose": (c_int, [c_void_p, c_i64, c_i64, c_void_p, c_void_p, c_i64, c_void_p]),
    "cb200_split_planes": (c_int, [c_void_p, c_void_p, c_i64, c_void_p, c_int, c_i64, c_void_p]),
    "cb200_dqn_td_targets": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_double, c_i64,
                                     c_i64, c_void_p, c_void_p, c_void_p]),
    "cb200_regression_head_loss_grad": (c_int, [c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_int, c_float, c_void_p,
                                                c_void_p, c_void_p]),
    "cb200_dqn_head_fused": (c_int, [c_void_p, c_void_p]),
    "cb200_ensemble_head_fused": (c_int, [c_void_p, c_void_p]),
    "cb200_nstep_q_head": (c_int, [c_void_p, c_void_p]),
    "cb200_actor_critic_head": (c_int, [c_void_p, c_void_p]),
    "cb200_actor_critic_gaussian_head": (c_int, [c_void_p, c_void_p]),
    "cb200_gaussian_policy_act": (c_int, [c_void_p, c_i64, ctypes.c_int32, c_void_p, c_void_p, c_void_p, c_void_p,
                                          c_void_p, c_void_p]),
    "cb200_categorical_act": (c_int, [c_void_p, c_i64, ctypes.c_int32, c_void_p, c_void_p, c_void_p, c_void_p]),
    "cb200_pg_targets": (c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_int32, c_i64, ctypes.c_int32, c_void_p,
                                 c_void_p, ctypes.c_int32, c_void_p, c_void_p, c_void_p, c_void_p]),
    "cb200_policy_gradient_head": (c_int, [c_void_p, c_void_p]),
    "cb200_policy_act": (c_int, [c_void_p, c_i64, ctypes.c_int32, ctypes.c_int32, c_void_p, c_void_p, c_void_p,
                                 c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "cb200_ensemble_action_values": (c_int, [c_void_p, c_i64, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32, c_void_p,
                                             c_float, c_void_p, c_void_p]),
    "cb200_dueling_combine_fwd": (c_int, [c_void_p, c_void_p, c_i64, c_i64, c_void_p, c_void_p]),
    "cb200_dueling_combine_bwd": (c_int, [c_void_p, c_i64, c_i64, c_void_p, c_void_p, c_void_p]),
    "cb200_sumsq": (c_int, [c_void_p, c_i64, c_void_p, c_void_p, c_void_p]),
    "cb200_clip_by_global_norm": (c_int, [c_void_p, c_i64, c_void_p, c_float, c_void_p]),
    "cb200_scale": (c_int, [c_void_p, c_i64, c_float, c_void_p]),
    "cb200_adam_tf": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_float, c_float, c_float, c_float,
                              c_float, c_float, c_void_p]),
    "cb200_adam_tf_dev": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_float, c_float, c_float, c_float,
                                  c_void_p, c_void_p]),
    "cb200_add_i64": (c_int, [c_void_p, c_i64, c_void_p]),
    "cb200_polyak": (c_int, [c_void_p, c_void_p, c_i64, c_double, c_void_p]),
    "cb200_ppo_continuous_head": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_i64,
                                          ctypes.c_int32, c_float, c_float, c_void_p, c_void_p, c_void_p, c_void_p]),
    "cb200_ppo_kl_head": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_i64, ctypes.c_int32,
                                  c_void_p, c_float, c_float, ctypes.c_int32, c_float, c_void_p, c_void_p, c_void_p,
                                  c_void_p]),
    "cb200_ppo_gaussian_act": (c_int, [c_void_p, c_void_p, c_i64, ctypes.c_int32, c_void_p, c_void_p, c_void_p,
                                       c_void_p]),
    "cb200_ppo_categorical_head": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_i64, ctypes.c_int32, c_float,
                                           c_void_p, c_float, c_void_p, c_void_p, c_void_p]),
    "cb200_gather_at": (c_int, [ctypes.POINTER(Column), c_int, c_void_p, c_void_p, c_i64, c_void_p]),
    "cb200_f64_to_f32": (c_int, [c_void_p, c_i64, c_void_p, c_void_p]),
    "cb200_sac_policy_sample": (c_int, [c_void_p, c_void_p, c_i64, ctypes.c_int32, c_void_p, c_void_p, c_void_p,
                                        c_void_p]),
    "cb200_sac_policy_grad": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_i64, ctypes.c_int32, c_void_p,
                                      c_void_p]),
    "cb200_sac_min_seed": (c_int, [c_void_p, c_void_p, c_i64, c_void_p, c_void_p, c_void_p, c_void_p]),
    "cb200_sub": (c_int, [c_void_p, c_void_p, c_i64, c_void_p, c_void_p]),
    "cb200_act_backward": (c_int, [c_void_p, ctypes.c_int32, c_void_p, ctypes.c_int32, c_i64, ctypes.c_int32,
                                   ctypes.c_int32, c_void_p, ctypes.c_int32, c_void_p]),
    "cb200_axpby_2d": (c_int, [c_void_p, ctypes.c_int32, c_i64, ctypes.c_int32, c_float, c_float, c_void_p,
                               ctypes.c_int32, c_void_p]),
    "cb200_ac_td_targets": (c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_int32, c_i64, c_double, ctypes.c_int32,
                                    ctypes.c_int32, c_double, c_double, c_void_p, c_void_p]),
    "cb200_naf_head": (c_int, [c_void_p, c_void_p]),
    "cb200_clip_by_value": (c_int, [c_void_p, c_i64, c_float, c_void_p]),
    "cb200_min2": (c_int, [c_void_p, c_void_p, c_i64, c_void_p, c_void_p]),
    "cb200_td3_smooth_actions": (c_int, [c_void_p, c_void_p, c_i64, c_double, c_double, c_double, c_void_p]),
    "cb200_c51_head": (c_int, [c_void_p] * 8 + [c_double, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32,
                               ctypes.c_int32] + [c_void_p] * 8),
    "cb200_c51_q_values": (c_int, [c_void_p, c_void_p, c_i64, ctypes.c_int32, c_void_p, c_void_p]),
    "cb200_qr_head": (c_int, [c_void_p, c_void_p]),
    "cb200_qr_q_values": (c_int, [c_void_p, c_i64, ctypes.c_int32, c_void_p, c_void_p]),
    "cb200_gae_scan": (c_int, [c_void_p, c_void_p, c_void_p, c_i64, c_double, c_double, c_void_p, c_void_p, c_void_p,
                               c_void_p]),
    "cb200_standardize": (c_int, [c_void_p, c_i64, c_void_p, c_void_p, c_void_p]),
    "cb200_nstep_returns": (c_int, [c_void_p, c_void_p, c_void_p, c_i64, c_double, c_i64, c_void_p, c_void_p]),
    "cb200_running_stats_push": (c_int, [c_void_p, c_i64, c_i64, c_void_p, c_void_p, c_void_p]),
    "cb200_running_stats_finalize": (c_int, [c_void_p, c_void_p, c_double, c_double, c_i64, c_void_p, c_void_p,
                                             c_void_p]),
    "cb200_running_stats_normalize": (c_int, [c_void_p, c_i64, c_i64, c_void_p, c_void_p, c_double, c_double,
                                              c_void_p, c_void_p, c_void_p]),
}

_lib = None


class CoachB200Error(RuntimeError):
    pass


def load():
    """Loads the library once; raises ImportError with build instructions when it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "coach_b200: %s is missing. The CUDA library is mandatory (there is no CPU path); build it with "
            "`python -m coach_b200.build`." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (restype, argtypes) in PROTOTYPES.items():
        fn = getattr(lib, name)      # AttributeError here = header / library mismatch: fail loudly
        fn.restype = restype
        fn.argtypes = argtypes
    if lib.cb200_abi_version() != 1:
        raise ImportError("coach_b200: ABI version mismatch between _lib.py and libcoach_b200.so")
    # CB200_TUNE_<KEY>=<int>: runtime knobs of the library (cb200_tune), e.g. CB200_TUNE_GEMM_TC=0 for A/B runs
    for k, v in os.environ.items():
        if k.startswith("CB200_TUNE_"):
            if lib.cb200_tune(k[len("CB200_TUNE_"):].lower().encode(), int(v)) != 0:
                raise ValueError("%s: %s" % (k, lib.cb200_last_error().decode("utf-8", "replace")))
    _lib = lib
    return lib


def check(rc):
    """Maps a C-ABI return code to the exception the reference would raise for the same condition."""
    if rc == 0:
        return
    msg = load().cb200_last_error().decode("utf-8", "replace")
    if rc == -1:
        raise ValueError(msg)
    raise CoachB200Error(msg)


def ptr(t):
    """Device/host pointer of a torch tensor (or None)."""
    return None if t is None else t.data_ptr()


def current_stream():
    import torch
    return torch.cuda.current_stream().cuda_stream


def make_columns(pairs):
    """pairs: iterable of (src_ptr, dst_ptr, row_bytes) -> (ctypes array, count)."""
    pairs = list(pairs)
    if len(pairs) > CB200_MAX_COLUMNS:
        raise ValueError("at most %d columns per call" % CB200_MAX_COLUMNS)
    arr = (Column * len(pairs))()
    for k, (s, d, rb) in enumerate(pairs):
        arr[k].src, arr[k].dst, arr[k].row_bytes = s, d, rb
    return arr, len(pairs)


def tune_default(name, default):
    """host-side feature switches: environment variable CB200_<NAME> overrides the default (benchmark A/B runs)"""
    v = os.environ.get("CB200_" + name.upper())
    return int(v) if v is not None else default
