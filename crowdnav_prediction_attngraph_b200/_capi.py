"""ctypes declarations of the C ABI in include/crowdnav_b200.h and the library loader.

The product path REQUIRES the compiled CUDA library (csrc/ -> libcrowdnav_b200.so, built in-tree
by `__graft_entry__.build()`); there is no Python or CPU fallback: a missing library raises.
"""
import ctypes as C
import os

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "libcrowdnav_b200.so")


class CnConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "num_envs", "nenv_total", "rank_offset", "seed", "human_num", "predict_steps", "const_vel",
        "randomize_attributes", "random_goal_changing", "end_goal_changing", "sort_humans", "device",
        "phase", "val_size", "test_size", "human_num_range", "human_policy")] + \
        [("robot_policy", C.c_int16), ("robot_visible", C.c_int16)] + \
        [(n, C.c_double) for n in (
            "time_step", "time_limit", "pred_timestep", "circle_radius", "arena_size",
            "discomfort_dist", "discomfort_penalty_factor", "success_reward", "collision_penalty",
            "human_radius", "human_v_pref", "human_fov", "robot_radius", "robot_v_pref", "robot_fov",
            "sensor_range", "goal_change_chance", "orca_neighbor_dist", "orca_safety_space",
            "orca_time_horizon", "sf_A", "sf_B", "sf_KI")]


class CnObsPtrs(C.Structure):
    _fields_ = [("robot_node", C.c_void_p), ("temporal_edges", C.c_void_p), ("spatial_edges", C.c_void_p),
                ("detected_human_num", C.c_void_p), ("visible_masks", C.c_void_p)]


class CnStepPtrs(C.Structure):
    _fields_ = [("reward", C.c_void_p), ("done", C.c_void_p), ("info", C.c_void_p), ("info_aux", C.c_void_p),
                ("ep_ret", C.c_void_p), ("ep_len", C.c_void_p), ("not_done", C.c_void_p)]


class CnCopySeg(C.Structure):
    _fields_ = [("dst", C.c_void_p), ("src", C.c_void_p), ("bytes", C.c_size_t)]


class CnPolicyConfig(C.Structure):
    _fields_ = [("num_envs", C.c_int32), ("human_num", C.c_int32), ("input_size", C.c_int32),
                ("device", C.c_int32), ("gemm_mode", C.c_int32)]


class CnActPtrs(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "robot_node", "temporal_edges", "spatial_edges", "detected_human_num", "h_in", "masks", "noise",
        "value", "action", "log_prob", "h_out", "action_mean")]


# every symbol include/crowdnav_b200.h declares (tests check the library exports all of them)
ABI_VERSION = 3          # include/crowdnav_b200.h CN_ABI_VERSION

EXPORTS = [
    "cn_last_error", "cn_abi_version", "cn_env_create", "cn_env_destroy", "cn_env_reset", "cn_env_step",
    "cn_env_step_host", "cn_env_state_bytes", "cn_env_state_copy", "cn_env_launch_count", "cn_env_profile", "cn_env_stage_ms",
    "cn_policy_create", "cn_policy_destroy", "cn_policy_set_param", "cn_policy_finalize",
    "cn_policy_act", "cn_policy_launch_count", "cn_policy_last_rows", "cn_policy_profile", "cn_policy_stage_count",
    "cn_policy_stage_name", "cn_policy_stage_ms", "cn_copy_segments", "cn_fetch_sync",
    "cn_gst_create", "cn_gst_destroy", "cn_gst_set_param", "cn_gst_finalize", "cn_gst_reset", "cn_gst_step",
    "cn_gst_launch_count",
    "cn_update_linear_saved_bytes", "cn_update_linear_ws_bytes", "cn_update_linear_fwd", "cn_update_linear_bwd",
    "cn_update_attn_fwd", "cn_update_attn_bwd", "cn_update_gru_fwd", "cn_update_gru_bwd",
]

_lib = None


def config_from_dict(d):
    cfg = CnConfig()
    for name, _ in CnConfig._fields_:
        setattr(cfg, name, d[name])
    return cfg


def default_config_dict(**over):
    """Defaults = the reference's crowd_nav/configs/config.py values for CrowdSimPred-v0/const_vel."""
    d = dict(
        num_envs=16, nenv_total=16, rank_offset=0, seed=425, human_num=20, predict_steps=5, const_vel=1,
        randomize_attributes=0, random_goal_changing=0, end_goal_changing=1, sort_humans=1, device=0,
        phase=0, val_size=100, test_size=500, human_num_range=0, human_policy=0, robot_policy=0, robot_visible=0,
        time_step=0.25, time_limit=50.0, pred_timestep=0.25, circle_radius=6 * 2 ** 0.5, arena_size=6.0,
        discomfort_dist=0.25, discomfort_penalty_factor=10.0, success_reward=10.0, collision_penalty=-20.0,
        human_radius=0.3, human_v_pref=1.0, human_fov=2.0, robot_radius=0.3, robot_v_pref=1.0, robot_fov=2.0,
        sensor_range=5.0, goal_change_chance=0.5, orca_neighbor_dist=10.0, orca_safety_space=0.15,
        orca_time_horizon=5.0, sf_A=2.0, sf_B=1.0, sf_KI=1.0)
    for k, v in over.items():
        if k not in d:
            raise TypeError("unknown config field %r" % k)
        d[k] = v
    return d


def load_library(path=None):
    """Load libcrowdnav_b200.so and declare prototypes.  Raises if it is missing."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or LIB_PATH
    if not os.path.exists(p):
        raise ImportError(
            "%s not found: build the CUDA extension first (python -c 'import __graft_entry__ as g; g.build()'). "
            "There is no CPU fallback." % p)
    lib = C.CDLL(p)
    lib.cn_last_error.restype = C.c_char_p
    lib.cn_abi_version.restype = C.c_int
    if lib.cn_abi_version() != ABI_VERSION:
        raise ImportError("%s has C ABI version %d, this package needs %d: rebuild the extension" % (
            p, lib.cn_abi_version(), ABI_VERSION))
    lib.cn_env_create.argtypes = [C.POINTER(CnConfig), C.POINTER(C.c_void_p)]
    lib.cn_env_destroy.argtypes = [C.c_void_p]
    lib.cn_env_reset.argtypes = [C.c_void_p, C.POINTER(CnObsPtrs), C.c_void_p]
    lib.cn_env_step.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(CnObsPtrs), C.POINTER(CnStepPtrs), C.c_void_p]
    lib.cn_env_step_host.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(CnObsPtrs), C.POINTER(CnStepPtrs)]
    lib.cn_env_state_bytes.restype = C.c_size_t
    lib.cn_env_state_bytes.argtypes = [C.c_void_p, C.c_char_p]
    lib.cn_env_state_copy.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_size_t, C.c_int]
    lib.cn_gst_create.restype = C.c_int
    lib.cn_gst_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_int, C.POINTER(C.c_void_p)]
    lib.cn_gst_destroy.argtypes = [C.c_void_p]
    lib.cn_gst_set_param.restype = C.c_int
    lib.cn_gst_set_param.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_size_t]
    lib.cn_gst_finalize.restype = C.c_int
    lib.cn_gst_finalize.argtypes = [C.c_void_p]
    lib.cn_gst_reset.restype = C.c_int
    lib.cn_gst_reset.argtypes = [C.c_void_p, C.c_void_p]
    lib.cn_gst_step.restype = C.c_int
    lib.cn_gst_step.argtypes = [C.c_void_p] * 7 + [C.c_void_p]
    lib.cn_gst_launch_count.restype = C.c_int64
    lib.cn_gst_launch_count.argtypes = [C.c_void_p]
    lib.cn_copy_segments.restype = C.c_int
    lib.cn_copy_segments.argtypes = [C.POINTER(CnCopySeg), C.c_int, C.c_int, C.c_void_p]
    lib.cn_fetch_sync.restype = C.c_int
    lib.cn_fetch_sync.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p]
    lib.cn_env_launch_count.restype = C.c_int64
    lib.cn_env_launch_count.argtypes = [C.c_void_p]
    lib.cn_env_profile.restype = C.c_int
    lib.cn_env_profile.argtypes = [C.c_void_p, C.c_int]
    lib.cn_env_stage_ms.restype = C.c_int
    lib.cn_env_stage_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
    lib.cn_policy_create.argtypes = [C.POINTER(CnPolicyConfig), C.POINTER(C.c_void_p)]
    lib.cn_policy_destroy.argtypes = [C.c_void_p]
    lib.cn_policy_set_param.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_size_t]
    lib.cn_policy_finalize.argtypes = [C.c_void_p, C.c_void_p]
    lib.cn_policy_act.argtypes = [C.c_void_p, C.POINTER(CnActPtrs), C.c_void_p]
    lib.cn_policy_launch_count.restype = C.c_int64
    lib.cn_policy_launch_count.argtypes = [C.c_void_p]
    lib.cn_policy_last_rows.restype = C.c_int64
    lib.cn_policy_last_rows.argtypes = [C.c_void_p]
    lib.cn_policy_profile.argtypes = [C.c_void_p, C.c_int]
    lib.cn_policy_stage_count.restype = C.c_int
    lib.cn_policy_stage_name.restype = C.c_char_p
    lib.cn_policy_stage_name.argtypes = [C.c_int]
    lib.cn_policy_stage_ms.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    lib.cn_update_linear_saved_bytes.restype = C.c_size_t
    lib.cn_update_linear_saved_bytes.argtypes = [C.c_int, C.c_int]
    lib.cn_update_linear_ws_bytes.restype = C.c_size_t
    lib.cn_update_linear_ws_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
    lib.cn_update_linear_fwd.argtypes = [C.c_void_p] * 6 + [C.c_size_t] + [C.c_int] * 5 + [C.c_void_p]
    lib.cn_update_linear_bwd.argtypes = [C.c_void_p] * 8 + [C.c_size_t] + [C.c_int] * 5 + [C.c_void_p]
    lib.cn_update_attn_fwd.argtypes = [C.c_void_p] * 3 + [C.c_int] + [C.c_void_p] * 2 + [C.c_int, C.c_void_p]
    lib.cn_update_attn_bwd.argtypes = [C.c_void_p] * 6 + [C.c_int] + [C.c_void_p] * 2 + [C.c_int, C.c_void_p]
    lib.cn_update_gru_fwd.argtypes = [C.c_void_p] * 5 + [C.c_int] * 2 + [C.c_void_p] * 2 + [C.c_int, C.c_void_p]
    lib.cn_update_gru_bwd.argtypes = [C.c_void_p] * 7 + [C.c_int] * 2 + [C.c_void_p] * 3 + [C.c_int, C.c_void_p]
    if path is None:
        _lib = lib
    return lib


def raw_stream(device_index):
    """The caller's current CUDA stream on that device as a c_void_p (torch's C-level query: ~0.3 us, where
    torch.cuda.current_stream(dev).cuda_stream costs ~7 us of Python per call)."""
    import torch
    return C.c_void_p(torch._C._cuda_getCurrentRawStream(device_index))


def check(lib, rc, what):
    if rc != 0:
        raise RuntimeError("%s failed: %s" % (what, lib.cn_last_error().decode()))
