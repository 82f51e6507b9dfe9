"""ctypes binding of the C ABI in include/b200ocl.h.  Fails loudly when the library
is missing -- there is no fallback path."""
import ctypes
import os
from ctypes import c_char_p, c_double, c_float, c_int, c_int64, c_size_t, c_uint64, c_void_p

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, 'libb200ocl.so')

P = c_void_p
# name -> (restype, argtypes); one entry per function declared in include/b200ocl.h
SIGNATURES = {
    'b200ocl_last_error': (c_char_p, []),
    'b200ocl_version': (c_int, []),
    'b200ocl_launch_count': (c_uint64, []),
    'b200ocl_sm_count': (c_int, []),
    'b200ocl_profile_begin': (None, []),
    'b200ocl_profile_end': (c_int, []),
    'b200ocl_profile_get': (c_int, [c_int, P, c_int, P, P, P]),
    'b200ocl_knn_sv_workspace_bytes': (c_size_t, [c_int, c_int, c_int]),
    'b200ocl_knn_sv': (c_int, [P, P, P, P, c_int, c_int, c_int, c_int, P, P, P, P, P, c_size_t, P]),
    'b200ocl_knn_sv_plan': (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, P]),
    'b200ocl_rank_desc': (c_int, [P, c_float, P, c_float, c_int, P, c_int, P, P]),
    'b200ocl_supcon_workspace_bytes': (c_size_t, [c_int, c_int, c_int]),
    'b200ocl_supcon': (c_int, [P, P, c_int, c_int, c_int, c_float, P, P, P, c_size_t, P]),
    'b200ocl_supcon_plan': (c_int, [c_int, c_int, c_int, c_int, c_int, P]),
    'b200ocl_gather_rows': (c_int, [P, P, c_int, c_size_t, P, P]),
    'b200ocl_scatter_rows': (c_int, [P, P, c_int, c_size_t, P, P]),
    'b200ocl_stream_prepare': (c_int, [P, P, c_int, c_int, c_int, P, P]),
    'b200ocl_stream_prepare_f64': (c_int, [P, P, c_int, c_int, c_int, P, P]),
    'b200ocl_ncm_class_means': (c_int, [P, P, c_int, c_int, P, c_int, P, P, P]),
    'b200ocl_ncm_classify': (c_int, [P, c_int, c_int, P, c_int, P, P, P, P, P]),
    'b200ocl_linear_argmax': (c_int, [P, c_int, c_int, P, P, c_int, P, P, P, P]),
    'b200ocl_linear_argmax_ea': (c_int, [P, c_int, c_int, P, P, c_int, P, P, P, P, P, P, P, P, P]),
    'b200ocl_rows_mean': (c_int, [P, P, c_int, c_int, P, c_int, P, P]),
    'b200ocl_cosine_argmax': (c_int, [P, c_int, c_int, P, c_int, P, P, P, P]),
    'b200ocl_linear_fwd': (c_int, [P, P, P, P, c_int, c_int, c_int, c_int, P]),
    'b200ocl_agem_project_workspace_bytes': (c_size_t, []),
    'b200ocl_agem_project': (c_int, [P, P, P, c_size_t, P, P, c_size_t, P]),
    'b200ocl_grad_cosine_workspace_bytes': (c_size_t, [c_int]),
    'b200ocl_grad_cosine': (c_int, [P, P, c_int, c_size_t, P, P, P, c_size_t, P]),
    'b200ocl_gem_project_workspace_bytes': (c_size_t, [c_int, c_size_t]),
    'b200ocl_gem_project': (c_int, [P, c_size_t, c_int, P, P, c_size_t, c_double, c_double, P, P, P, P, P, c_size_t,
                                    P]),
    'b200ocl_gem_plan': (c_int, [c_int, c_size_t, c_int, P]),
    'b200ocl_sgd_step': (c_int, [P, P, P, c_size_t, c_float, c_float, P]),
    # ResNet engine: descriptor / state / info structs are passed by pointer (see engine.py)
    'b200ocl_net_query': (c_int, [P, P]),
    'b200ocl_net_tensor': (c_int, [P, c_int, P, P, P]),
    'b200ocl_net_pack': (c_int, [P, P, P]),
    'b200ocl_net_eval_workspace_bytes': (c_size_t, [P, c_int]),
    'b200ocl_net_features_eval': (c_int, [P, P, P, c_int, P, P, c_size_t, P]),
    'b200ocl_net_train_workspace_bytes': (c_size_t, [P, c_int]),
    'b200ocl_net_train_ws_layout': (c_int, [P, c_int, c_int, P]),
    'b200ocl_net_conv_geom': (c_int, [P, c_int, c_int, c_int, c_int, P]),
    'b200ocl_net_forward_train': (c_int, [P, P, P, c_int, P, P, c_size_t, P]),
    'b200ocl_net_forward_evalgrad': (c_int, [P, P, P, c_int, P, P, c_size_t, P]),
    'b200ocl_net_forward_train_deferred': (c_int, [P, P, P, c_int, P, P, c_size_t, P]),
    'b200ocl_net_apply_running_stats': (c_int, [P, P, c_int, P, c_size_t, P]),
    'b200ocl_net_backward': (c_int, [P, P, P, P, c_int, P, c_size_t, c_int, P]),
    'b200ocl_net_sgd_step': (c_int, [P, P, c_float, c_float, P, P]),
    'b200ocl_net_sgd_step_clipped_workspace_bytes': (c_size_t, [P]),
    'b200ocl_net_sgd_step_clipped': (c_int, [P, P, c_float, c_float, c_float, P, P, c_size_t, P]),
    'b200ocl_net_sgd_step_ewc_workspace_bytes': (c_size_t, [P]),
    'b200ocl_net_sgd_step_ewc': (c_int, [P, P, P, c_float, c_float, c_float, c_int, c_float, c_float, P, P, c_size_t,
                                         P]),
    'b200ocl_adam_step': (c_int, [P, P, P, P, c_size_t, P, c_int, P]),
    'b200ocl_net_adam_step': (c_int, [P, P, P, P, c_int, P]),
    'b200ocl_net_adam_step_ewc': (c_int, [P, P, P, P, P, c_int, c_float, c_int, c_float, c_float, P, P, c_size_t, P]),
    'b200ocl_ewc_consolidate_workspace_bytes': (c_size_t, [P]),
    'b200ocl_ewc_consolidate': (c_int, [P, P, P, P, c_size_t, P]),
    'b200ocl_ce_loss': (c_int, [P, P, c_int, c_int, P, P, P, P, P, P]),
    'b200ocl_cls_loss': (c_int, [P, P, c_int, c_int, c_int, P, c_int, c_int, P, c_int, P, c_float, c_float, P, P, P, P,
                                 P]),
    'b200ocl_icarl_loss': (c_int, [P, P, P, P, c_int, c_int, c_int, c_int, c_int, c_int, P, P, P, P]),
    'b200ocl_logit_mse': (c_int, [P, P, c_int, P, c_int, c_int, c_double, P, P, P, P]),
    'b200ocl_pcr_loss_workspace_bytes': (c_size_t, [c_int, c_int]),
    'b200ocl_pcr_loss': (c_int, [P, P, c_int, c_int, P, c_int, c_float, P, P, P, P, P, P, c_size_t, P]),
    'b200ocl_scr_augment': (c_int, [P, P, P, c_int, c_int, c_int, P]),
    'b200ocl_aser_replace': (c_int, [P, c_int, c_int, P, P, P, c_int, c_size_t, P, P, P, P]),
    'b200ocl_conv_selftest_workspace_bytes': (c_size_t, [c_int, c_int, c_int, c_int, c_int, c_int, c_int]),
    'b200ocl_conv_selftest_geom': (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                           P]),
    'b200ocl_conv_selftest': (c_int, [P, P, P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, P, P, c_size_t, P]),
    'b200ocl_conv_selftest_eval': (c_int, [P, P, P, P, c_int, P, c_int, c_int, c_int, c_int, c_int, P, c_size_t, P]),
    'b200ocl_selftest_umma_tf32': (c_int, [P, P, P, c_int, c_int, c_int, P, P]),
    'b200ocl_selftest_umma_window': (c_int, [P, P, P, c_int, c_int, c_int, c_int, c_int, P, P]),
    'b200ocl_wgrad_tc_selftest_workspace_bytes': (c_size_t, [c_int, c_int, c_int, c_int, c_int]),
    'b200ocl_wgrad_tc_selftest_geom': (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, P]),
    'b200ocl_wgrad_tc_selftest': (c_int, [P, P, P, c_int, c_int, c_int, c_int, c_int, P, c_size_t, P]),
    'b200ocl_snapshot_workspace_bytes': (c_size_t, [c_int]),
    'b200ocl_snapshot_pack': (c_int, [P, c_int, P, c_size_t, P, c_size_t, P]),
    'b200ocl_snapshot_unpack': (c_int, [P, c_int, P, c_size_t, P, c_size_t, P]),
}

_lib = None

# The library is built for sm_90a only; no such part has more SMs than the H100 SXM's 132.
MAX_SMS = 132


class NativeError(RuntimeError):
    pass


def parse_sm_count(text, device_sms):
    """The SM count B200OCL_SM_COUNT asks the library to plan for, or None when it is unset (text None).  Refuses
    anything but an integer in [1, device_sms]: a grid planned for more SMs than the device has could leave part of a
    grid-synchronised kernel (fused BN backward, fused SupCon) waiting for CTAs that never get an SM."""
    if text is None:
        return None
    try:
        n = int(text.strip())
    except ValueError:
        raise ValueError('B200OCL_SM_COUNT=%r is not an integer' % text) from None
    if not 1 <= n <= device_sms:
        raise ValueError('B200OCL_SM_COUNT=%d is outside [1, %d], the SM counts this device can run' % (n, device_sms))
    return n


def _device_sms():
    """The fewest SMs of any visible device; MAX_SMS where there is none."""
    import torch
    if not torch.cuda.is_available():
        return MAX_SMS
    return min(torch.cuda.get_device_properties(i).multi_processor_count for i in range(torch.cuda.device_count()))


def lib():
    global _lib
    if _lib is None:
        if os.environ.get('B200OCL_SM_COUNT') is not None:
            parse_sm_count(os.environ['B200OCL_SM_COUNT'], _device_sms())
        if not os.path.exists(LIB_PATH):
            raise NativeError('%s is missing: build it with `python __graft_entry__.py` (nvcc, sm_90a). '
                              'b200ocl has no CPU or library fallback.' % LIB_PATH)
        handle = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def check(rc, what):
    if rc != 0:
        msg = lib().b200ocl_last_error()
        raise NativeError('%s failed (code %d): %s' % (what, rc, msg.decode() if msg else '?'))


def launch_count():
    return int(lib().b200ocl_launch_count())
