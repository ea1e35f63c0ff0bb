"""ctypes binding of libspo.so (the C-ABI declared in include/spo.h).

PyTorch is used only as the owner of device memory and streams: every call passes
``tensor.data_ptr()`` and the current CUDA stream handle.  There is no fallback: if the
shared library is missing or a call fails, a ``SpoError`` is raised.
"""
from __future__ import annotations

import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libspo.so")


class SpoError(RuntimeError):
    pass


class Dims(C.Structure):
    _fields_ = [("obs_dim", C.c_int), ("act_dim", C.c_int), ("hidden", C.c_int)]


_fp = C.c_void_p


class Rollout(C.Structure):
    _fields_ = [("obs", _fp), ("act", _fp), ("reward", _fp), ("cost", _fp), ("value_r", _fp), ("value_c", _fp),
                ("logp", _fp), ("seg_end", _fp), ("boot_r", _fp), ("boot_c", _fp),
                ("num_envs", C.c_int), ("steps", C.c_int)]


class Batch(C.Structure):
    _fields_ = [("obs", _fp), ("act", _fp), ("logp", _fp), ("target_r", _fp), ("target_c", _fp), ("adv", _fp),
                ("old_mean", _fp), ("old_std", _fp), ("count", C.c_int64)]


class HParams(C.Structure):
    _fields_ = [("lr_actor", C.c_float), ("lr_reward", C.c_float), ("lr_cost", C.c_float),
                ("beta1", C.c_float), ("beta2", C.c_float), ("adam_eps", C.c_float),
                ("max_grad_norm", C.c_float), ("critic_l2", C.c_float),
                ("clip_lo", C.c_float), ("clip_hi", C.c_float),
                ("focops_lam", C.c_float), ("focops_kl", C.c_float), ("value_coef", C.c_float)]


class Comm(C.Structure):
    _fields_ = [("world", C.c_int), ("rank", C.c_int), ("grad_bufs", C.c_void_p), ("flags", C.c_void_p),
                ("seq_base", C.c_ulonglong), ("spin_limit", C.c_uint)]


# numpy view of spo_update_ctrl (64 bytes): see include/spo.h
CTRL_BYTES = 64
CTRL_DTYPE = [("loss_sum", "<f8", 3), ("kl_sum", "<f8"), ("steps", "<i8"), ("stop", "<i4"), ("passes", "<i4"),
              ("final_kl", "<f4"), ("ticket", "<u4"), ("extra_sumsq", "<f4"), ("pad", "<i4")]
CTRL_EXTRA_SUMSQ_F32_INDEX = 14  # byte offset 56
CTRL_KL_SUM_F64_INDEX = 3        # byte offset 24

LOSS_PPO_CLIP, LOSS_FOCOPS, LOSS_CRITIC_ONLY, LOSS_PG, LOSS_CUP_PROJECTION = 0, 1, 2, 3, 4
MA_RATIO_PRODUCT, MA_RATIO_PER_DIM = 0, 1       # ratio_mode of spo_ma_ppo_actor_loss / _finalize

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise SpoError(f"{LIB_PATH} not found: build it with `python safe-policy-optimization_b200/build.py` "
                           "(there is no CPU / PyTorch fallback for the hot path)")
        _lib = C.CDLL(LIB_PATH)
        _lib.spo_last_error.restype = C.c_char_p
        _declare(_lib)
    return _lib


def _declare(L):
    i, i64, f, d, u64, p = C.c_int, C.c_int64, C.c_float, C.c_double, C.c_uint64, C.c_void_p
    PD = C.POINTER(Dims)
    sig = {
        "spo_version": [],
        "spo_sync_check": [p],
        "spo_param_count": [PD, C.POINTER(i), C.POINTER(i), C.POINTER(i)],
        "spo_param_offsets": [PD, i] + [C.POINTER(i)] * 7,
        "spo_policy_step": [PD, p, p, p, u64, u64, i, i, p, p, p, p, C.POINTER(Rollout), i, p],
        "spo_critic_values": [PD, p, p, i, p, p, p],
        "spo_store_transition": [C.POINTER(Rollout), i, p, p, p, p, i, p, p, p, p, p],
        "spo_gae_dual": [p, p, p, p, p, p, p, f, d, d, p, p, p, p, i, i, i, p],
        "spo_adv_stats": [p, p, i64, p, p],
        "spo_adv_apply": [p, p, i64, p, i, i, f, f, p, p],
        "spo_pg_update": [PD, p, p, p, p, C.POINTER(Batch), p, i64, i, i, C.POINTER(HParams), p, p],
        "spo_comm_slot_floats": [PD, C.POINTER(i)],
        "spo_pg_update_dp": [PD, p, p, p, p, C.POINTER(Batch), p, i64, i, i, C.POINTER(HParams), p, C.POINTER(Comm), p],
        "spo_comm_alloc": [C.c_size_t, C.POINTER(p)],
        "spo_comm_free": [p],
        "spo_comm_export": [p, C.c_char_p],
        "spo_comm_import": [C.c_char_p, C.POINTER(p)],
        "spo_comm_close": [p],
        "spo_actor_kl_accumulate": [PD, p, p, p, p, i64, p, p],
        "spo_kl_finalize": [p, d, f, p],
        "spo_actor_forward": [PD, p, p, i64, p, p],
        "spo_actor_kl": [PD, p, p, p, p, i64, i, f, p, p],
        "spo_surrogate_grad": [PD, p, p, p, p, p, i64, p, p, p],
        "spo_fvp": [PD, p, p, i64, p, f, p, p],
        "spo_linesearch_eval": [PD, p, p, p, p, p, p, p, p, i64, p, p],
        "spo_conjugate_gradient": [PD, p, p, i64, p, i, f, f, f, p, p, p],
        "spo_ma_mlp_layer": [p, i, i, p, p, p, p, i, p, p, p, p],
        "spo_ma_head": [p, i, i, p, p, i, p, f, f, p, p, p, p],
        "spo_ma_mlp_layer_train": [p, i, i, p, p, p, p, i, p, p, p, p, p, p],
        "spo_ma_ln_elu_bwd": [p, p, p, i, i, p, p, p],
        "spo_ma_ln_in_bwd": [p, p, i, i, p, p],
        "spo_ma_partial_reduce": [p, i, i, i, i, p, p, p, f, p],
        "spo_ma_gemm_nn": [p, p, p, i, i, i, p],
        "spo_ma_gemm_tn": [p, p, p, i, i, i, i, p],
        "spo_ma_actor_loss": [p, i, i, p, p, p, i, p, p, p, p, p, p, f, f, f, f, p, p, p, p],
        "spo_ma_actor_finalize": [p, i, i, p, i, f, f, f, p, p, p, p],
        "spo_ma_value_loss": [p, p, p, p, i, f, f, f, p, p, p],
        "spo_ma_popart_normalize": [p, i, p, d, f, p, p],
        "spo_ma_lagrange_step": [p, p, p, i, f, d, f, p, p],
        "spo_ma_clip_adam": [p, p, p, p, i, f, d, d, d, d, d, i, p, p, p],
        "spo_ma_mlp_layer_jvp": [p, p, i, i, p, p, p, p, p, p, p, i, p, p, p, p, p, p],
        "spo_ma_head_jvp": [p, p, i, i, p, p, p, i, p, f, f, p, p, p],
        "spo_ma_fvp_finalize": [p, p, p, i, p, i, i, f, f, f, p],
        "spo_ma_ratio_loss": [p, i, p, i, p, p, p, p, f, f, f, p, p, p],
        "spo_ma_work_floats": [],
        "spo_ma_dots": [p, p, p, p, p, p, p, p, i, i, p, p, p],
        "spo_ma_cg_begin": [p, p, p, p, i, p, p, p],
        "spo_ma_cg_update": [p, p, p, p, i, f, p, p, p],
        "spo_ma_step_dir": [p, p, f, f, i, p, i, p],
        "spo_ma_ls_trial": [p, p, p, f, p, i, p],
        "spo_ma_linesearch_eval": [p, p, p, p, i, p, p, p, p, p, i, f, f, p, p, p],
        "spo_ma_ppo_actor_loss": [p, i, i, p, p, p, i, p, p, p, p, p, p, p, p, i, f, f, f, f, p, p, p, p],
        "spo_ma_ppo_actor_finalize": [p, i, i, p, i, p, i, f, f, f, p, p, p, p],
        "spo_ma_value_loss_masked": [p, p, p, p, p, p, i, f, f, f, p, p, p],
        "spo_cg_begin": [PD, p, p, p, p],
        "spo_cg_update": [PD, p, p, f, f, p],
        "spo_obs_normalize": [p, i, i, p, p, d, p, i, d, p, p],
        "spo_action_rescale": [p, i, i, p, p, f, f, p, p],
        "spo_gae_masked": [p, p, p, f, f, f, d, p, i, i, p],
    }
    for name, args in sig.items():
        fn = getattr(L, name)
        fn.argtypes = args
        fn.restype = C.c_int


EXPORTS = ("spo_version", "spo_last_error", "spo_sync_check", "spo_param_count", "spo_param_offsets",
           "spo_policy_step", "spo_critic_values", "spo_store_transition", "spo_gae_dual", "spo_adv_stats",
           "spo_adv_apply", "spo_pg_update", "spo_actor_forward", "spo_actor_kl", "spo_surrogate_grad", "spo_fvp",
           "spo_linesearch_eval", "spo_conjugate_gradient", "spo_comm_slot_floats", "spo_pg_update_dp", "spo_comm_alloc",
           "spo_comm_free", "spo_comm_export", "spo_comm_import", "spo_comm_close", "spo_actor_kl_accumulate", "spo_kl_finalize",
           "spo_obs_normalize", "spo_action_rescale", "spo_gae_masked", "spo_cg_begin", "spo_cg_update", "spo_ma_mlp_layer", "spo_ma_head",
           "spo_ma_mlp_layer_train", "spo_ma_ln_elu_bwd", "spo_ma_ln_in_bwd", "spo_ma_partial_reduce", "spo_ma_gemm_nn", "spo_ma_gemm_tn", "spo_ma_actor_loss", "spo_ma_actor_finalize", "spo_ma_value_loss", "spo_ma_popart_normalize", "spo_ma_lagrange_step", "spo_ma_clip_adam",
           "spo_ma_work_floats", "spo_ma_mlp_layer_jvp", "spo_ma_head_jvp", "spo_ma_fvp_finalize", "spo_ma_ratio_loss", "spo_ma_dots", "spo_ma_cg_begin", "spo_ma_cg_update", "spo_ma_step_dir", "spo_ma_ls_trial", "spo_ma_linesearch_eval",
           "spo_ma_ppo_actor_loss", "spo_ma_ppo_actor_finalize", "spo_ma_value_loss_masked")


# number of libspo kernels launched so far (bench.py reports the delta over its timed region)
LAUNCHES = {"n": 0}
_KERNEL_CALLS = {"spo_policy_step", "spo_critic_values", "spo_store_transition", "spo_gae_dual", "spo_adv_stats",
                 "spo_adv_apply", "spo_pg_update", "spo_actor_forward", "spo_actor_kl", "spo_surrogate_grad", "spo_fvp",
                 "spo_linesearch_eval", "spo_pg_update_dp", "spo_actor_kl_accumulate", "spo_kl_finalize", "spo_obs_normalize",
                 "spo_action_rescale", "spo_gae_masked", "spo_cg_begin", "spo_cg_update", "spo_ma_mlp_layer", "spo_ma_head",
                 "spo_ma_mlp_layer_train", "spo_ma_ln_elu_bwd", "spo_ma_ln_in_bwd", "spo_ma_partial_reduce", "spo_ma_gemm_nn", "spo_ma_gemm_tn", "spo_ma_actor_loss", "spo_ma_actor_finalize", "spo_ma_value_loss", "spo_ma_popart_normalize", "spo_ma_lagrange_step", "spo_ma_clip_adam",
                 "spo_ma_mlp_layer_jvp", "spo_ma_head_jvp", "spo_ma_fvp_finalize", "spo_ma_ratio_loss", "spo_ma_dots", "spo_ma_cg_begin", "spo_ma_cg_update", "spo_ma_step_dir", "spo_ma_ls_trial", "spo_ma_linesearch_eval",
                 "spo_ma_ppo_actor_loss", "spo_ma_ppo_actor_finalize", "spo_ma_value_loss_masked"}


def check(rc, what):
    if what in _KERNEL_CALLS:
        LAUNCHES["n"] += 1
    if rc != 0:
        raise SpoError(f"{what} failed ({rc}): {lib().spo_last_error().decode()}")


def ptr(t):
    """Device pointer of a tensor (None -> NULL).  Tensors must be contiguous CUDA tensors."""
    if t is None:
        return None
    if not t.is_cuda:
        raise SpoError("libspo needs CUDA tensors (no CPU fallback)")
    if not t.is_contiguous():
        raise SpoError("libspo needs contiguous tensors")
    return t.data_ptr()


def stream():
    return torch.cuda.current_stream().cuda_stream


def dims(obs_dim, act_dim, hidden=64):
    return Dims(int(obs_dim), int(act_dim), int(hidden))


def param_count(d):
    a, c, t = C.c_int(), C.c_int(), C.c_int()
    check(lib().spo_param_count(C.byref(d), C.byref(a), C.byref(c), C.byref(t)), "spo_param_count")
    return a.value, c.value, t.value


def param_offsets(d, net):
    out = [C.c_int() for _ in range(7)]
    check(lib().spo_param_offsets(C.byref(d), net, *[C.byref(o) for o in out]), "spo_param_offsets")
    return dict(zip(("log_std", "w1", "b1", "w2", "b2", "w3", "b3"), (o.value for o in out)))
