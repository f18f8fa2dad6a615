"""ctypes binding of libdvd_b200.so (C ABI declared in include/dvd_b200.h).

The library is mandatory: importing the compute ops without it raises — there is no CPU or
PyTorch fallback on the product path.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libdvd_b200.so')

c_f32p = ctypes.c_void_p


class LossCfg(ctypes.Structure):
    """struct dvd_loss_cfg (include/dvd_b200.h)."""
    _fields_ = [('midas', ctypes.c_int), ('warm', ctypes.c_int), ('disp_mode', ctypes.c_int),
                ('second_is_disp', ctypes.c_int), ('flow_mul', ctypes.c_float), ('disp_mul', ctypes.c_float)]


DVD_CONV_MAX_TAPS = 128


class ConvDesc(ctypes.Structure):
    """struct dvd_conv_desc (include/dvd_b200.h)."""
    _fields_ = [('N', ctypes.c_int), ('H', ctypes.c_int), ('W', ctypes.c_int), ('Cin', ctypes.c_int),
                ('OH', ctypes.c_int), ('OW', ctypes.c_int), ('Cout', ctypes.c_int), ('stride', ctypes.c_int),
                ('ntaps', ctypes.c_int), ('kblock', ctypes.c_int), ('YH', ctypes.c_int), ('YW', ctypes.c_int),
                ('oy_mul', ctypes.c_int), ('oy_add', ctypes.c_int), ('ox_mul', ctypes.c_int), ('ox_add', ctypes.c_int),
                ('relu', ctypes.c_int), ('round_out', ctypes.c_int), ('bn_eps', ctypes.c_float),
                ('dy', ctypes.c_byte * DVD_CONV_MAX_TAPS), ('dx', ctypes.c_byte * DVD_CONV_MAX_TAPS),
                ('wt', ctypes.c_ubyte * DVD_CONV_MAX_TAPS)]


class PackItem(ctypes.Structure):
    """struct dvd_pack_item (include/dvd_b200.h)."""
    _fields_ = [('weight', ctypes.c_void_p), ('w_fwd', ctypes.c_void_p), ('w_bwd', ctypes.c_void_p), ('bn_gamma', ctypes.c_void_p),
                ('bn_var', ctypes.c_void_p), ('s_co', ctypes.c_long), ('s_ci', ctypes.c_long), ('s_ky', ctypes.c_long),
                ('s_kx', ctypes.c_long), ('blk0', ctypes.c_long), ('Cout', ctypes.c_int), ('Cin', ctypes.c_int),
                ('ksize', ctypes.c_int), ('groups', ctypes.c_int), ('kblock', ctypes.c_int), ('bn_eps', ctypes.c_float)]


DVD_MLP_MAX_NIN = 256
DVD_MLP_MAX_FREQ_XYZ = 42
DVD_MLP_MAX_FREQ_T = 126


class MlpCfg(ctypes.Structure):
    """struct dvd_mlp_cfg (include/dvd_b200.h)."""
    _fields_ = [('n_freq_xyz', ctypes.c_int), ('n_freq_t', ctypes.c_int), ('time_dependent', ctypes.c_int),
                ('sf_mag_div', ctypes.c_float), ('freq_xyz', ctypes.c_float * DVD_MLP_MAX_FREQ_XYZ),
                ('freq_t', ctypes.c_float * DVD_MLP_MAX_FREQ_T)]


_I, _F, _P = ctypes.c_int, ctypes.c_float, ctypes.c_void_p
_L = ctypes.c_longlong

# name -> argtypes; restype is int unless listed in _RESTYPES
SIGNATURES = {
    'dvd_version': [],
    'dvd_struct_size': [_I],
    'dvd_last_error': [],
    'dvd_reproject_partials_size': [_I, _I, _I],
    'dvd_unproject_fwd': [_P, _P, _P, _I, _I, _I, _I, _P],
    'dvd_unproject_bwd': [_P, _P, _P, _I, _I, _I, _I, _P],
    'dvd_reproject_loss_fwd': [_P, _P, _P, _P, _P, _P, ctypes.POINTER(LossCfg), _P, _P, _I, _I, _I, _P],
    'dvd_reproject_loss_bwd': [_P, _P, _P, _P, _P, _P, ctypes.POINTER(LossCfg), _P, _F, _P, _P, _P, _I, _I, _I, _P],
    'dvd_reproject_materialize': [_P] * 14 + [_I, _I, _I, _P],
    'dvd_reproject_materialize_bwd': [_P] * 17 + [_I, _I, _I, _P],
    'dvd_selftest_umma': [_P, _P, _P, _I, _I, _I, _I, _P],
    'dvd_mlp_packed_weights_bytes': [ctypes.POINTER(MlpCfg)],
    'dvd_mlp_save_bytes_per_eval': [ctypes.POINTER(MlpCfg), ctypes.c_long],
    'dvd_mlp_dy_bytes': [ctypes.POINTER(MlpCfg), ctypes.c_long],
    'dvd_mlp_pack_weights': [ctypes.POINTER(MlpCfg), ctypes.POINTER(ctypes.c_void_p), _P, _P, _P],
    'dvd_mlp_chain_fwd': [ctypes.POINTER(MlpCfg), _P, _P, _P, _P, _F, _I, _I, _P, _P, _P, _P,
                          ctypes.c_long, ctypes.c_long, _P],
    'dvd_mlp_dgrad': [ctypes.POINTER(MlpCfg), _P, _P, _P, _F, _I, _I, _P, _P, _P, _P, _P, _P, _P,
                      ctypes.c_long, ctypes.c_long, _P],
    'dvd_mlp_wgrad': [ctypes.POINTER(MlpCfg), _P, _P, ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(ctypes.c_void_p),
                      ctypes.c_long, _P],
    'dvd_acc_reg': [_P, _P, _F, _F, _P, _P, _P, _P, ctypes.c_long, _P],
    'dvd_adam_flat': [_P, _P, _P, _P, ctypes.c_long, _F, _F, _F, _F, _I, _F, _P],
    'dvd_adam_flat_dev': [_P, _P, _P, _P, ctypes.c_long, _F, _F, _F, _F, _P, _F, _P],
    'dvd_bn_act_fwd': [_P, _P, _P, _P, _P, _P, _F, _P, ctypes.c_long, _I, _I, _P],
    'dvd_bn_act_bwd': [_P, _P, _P, _P, _P, _P, _F, _P, _P, _P, _P, ctypes.c_long, _I, _I, _P],
    'dvd_upsample2x_fwd': [_P, _P, _I, _I, _I, _I, _I, _I, _P],
    'dvd_upsample2x_bwd': [_P, _P, _I, _I, _I, _I, _I, _I, _P],
    'dvd_conv2d_nhwc': [ctypes.POINTER(ConvDesc)] + [_P] * 11 + [_P],
    'dvd_conv2d_nhwc_ws': [ctypes.POINTER(ConvDesc)] + [_P] * 11 + [_P, ctypes.c_size_t, _P],
    'dvd_conv2d_workspace_bytes': [],
    'dvd_conv2d_streamk_bounds': [_I, _I, _I, ctypes.POINTER(ctypes.c_long)],
    'dvd_conv2d_pack': [_P, ctypes.c_long, ctypes.c_long, ctypes.c_long, ctypes.c_long, _P, _P, _I, _I, _I, _I, _I, _P, _P, _F, _P],
    'dvd_conv2d_pack_blocks': [_I, _I, _I, _I, _I],
    'dvd_conv2d_pack_batch': [_P, _I, ctypes.c_long, _I, _P],
    'dvd_conv2d_wgrad': [ctypes.POINTER(ConvDesc), _P, _P, _P, _P, ctypes.c_long, ctypes.c_long, ctypes.c_long, ctypes.c_long,
                         _I, _I, _P, _P, _P, _P, _P, _P],
    'dvd_conv2d_cluster_info': [ctypes.POINTER(ctypes.c_int)],
    'dvd_round_tf32': [_P, _P, ctypes.c_long, _P],
    'dvd_relu_bwd_colsum': [_P, _P, _P, _P, _P, _P, _F, _P, ctypes.c_long, _I, _I, _P],
    'dvd_maxpool3x3s2_fwd': [_P, _P, _P, _I, _I, _I, _I, _P],
    'dvd_maxpool3x3s2_bwd': [_P, _P, _P, _I, _I, _I, _I, _P],
    'dvd_stem_fwd': [_P, _P, ctypes.c_long, ctypes.c_long, ctypes.c_long, ctypes.c_long, _P, _P, _P, _P, _F,
                     ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float), _P, _I, _I, _I, _I, _P],
    'dvd_stem_wgrad': [_P, _P, _P, _P, _P, ctypes.c_long, ctypes.c_long, ctypes.c_long, ctypes.c_long, _P, _P, _P, _F, _P, _P,
                       ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float), _P, _I, _I, _I, _P],
    'dvd_head_fwd': [_P, _P, _P, _P, ctypes.c_long, _P],
    'dvd_head_bwd': [_P, _P, _P, _P, _P, _P, _P, ctypes.c_long, _I, _I, _P],
    'dvd_flow_resize_cubic': [_P, ctypes.c_size_t, _P, ctypes.c_size_t, _I, _I, _I, _I, _I, _P],
    'dvd_flow_pair_masks': [_P, _P, ctypes.c_size_t, _P, _P, ctypes.c_size_t, _I, _I, _I, _I, _P],
    'dvd_disp_vali_partials_size': [_I, _I, _I],
    'dvd_disp_vali': [_P, _P, _P, _P, _P, _I, _I, _I, _P],
    'dvd_raft_stem_fwd': [_P, _P, _P, _P, ctypes.c_size_t, _I, _I, _I, _P],
    'dvd_raft_instnorm_scratch_bytes': [_I, _I],
    'dvd_raft_instnorm_stats': [_P, _P, _P, ctypes.c_size_t, _I, ctypes.c_long, _I, _F, _P],
    'dvd_raft_norm_act': [_P, _P, _P, _P, _I, ctypes.c_long, _I, _I, _I, _I, _P],
    'dvd_raft_pyramid_floats': [_I, _I, _I],
    'dvd_raft_corr_pyramid': [_P, _P, _P, ctypes.c_size_t, _I, _I, _I, _I, _P],
    'dvd_raft_lookup': [_P, ctypes.c_size_t, _P, _P, ctypes.c_size_t, _I, _I, _I, _I, _P],
    'dvd_raft_convf1': [_P, _P, _P, _P, _I, _I, _I, _I, _P],
    'dvd_raft_context_split': [_P, _P, _P, _P, ctypes.c_long, _P],
    'dvd_raft_motion_pack': [_P, _P, _P, _P, _I, _I, _I, _P],
    'dvd_raft_gru_rh': [_P, _P, _P, ctypes.c_long, _P],
    'dvd_raft_gru_update': [_P, _P, _P, _P, _P, ctypes.c_long, _P],
    'dvd_raft_flow_head': [_P, _P, _P, _P, _P, _I, _I, _I, _P],
    'dvd_raft_upsample': [_P, _P, _P, _P, _P, ctypes.c_size_t, _I, _I, _I, _F, _P],
}
DVD_MASKS_FLOWPAIR_U8 = 0
DVD_MASKS_PAIRFILE_F32 = 1
_RESTYPES = {'dvd_last_error': ctypes.c_char_p, 'dvd_struct_size': ctypes.c_long, 'dvd_conv2d_workspace_bytes': ctypes.c_size_t, 'dvd_conv2d_pack_blocks': ctypes.c_long, 'dvd_mlp_packed_weights_bytes': ctypes.c_size_t,
             'dvd_mlp_save_bytes_per_eval': ctypes.c_size_t, 'dvd_mlp_dy_bytes': ctypes.c_size_t,
             'dvd_raft_instnorm_scratch_bytes': ctypes.c_long, 'dvd_raft_pyramid_floats': ctypes.c_long}

_lib = None


def load():
    """Load (once) and return the ctypes handle; raises RuntimeError if the .so is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            'libdvd_b200.so not found at %s — build it with `python -c "import __graft_entry__ as g; g.build()"` '
            '(or dynamic-video-depth_b200/csrc/build.sh). dvd_b200 has no CPU fallback.' % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is missing: fail loudly
        fn.argtypes = argtypes
        fn.restype = _RESTYPES.get(name, ctypes.c_int)
    _lib = lib
    return lib


def check(rc, what):
    if rc != 0:
        msg = load().dvd_last_error()
        raise RuntimeError('%s failed (rc=%d): %s' % (what, rc, (msg or b'').decode()))
