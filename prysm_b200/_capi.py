"""ctypes binding of libprysm_b200.so (the C ABI declared in include/prysm_b200.h).

The library is dlopen'ed directly -- no pybind / torch-extension layer.  If it is missing the
import fails loudly: there is no CPU or PyTorch fallback anywhere in this package.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, '_lib', 'libprysm_b200.so')

PB_C64, PB_C128 = 0, 1
ELEM_F32, ELEM_F64, ELEM_C64, ELEM_C128, ELEM_U8, ELEM_U16, ELEM_U32, ELEM_I32, ELEM_I64 = range(9)
IN_COMPLEX, IN_REAL, IN_AMP_OPD = 0, 1, 2
AMP_NONE, AMP_REAL, AMP_U8 = 0, 1, 2
OUT_COMPLEX, OUT_INTENSITY, OUT_ACCUMULATE = 0, 1, 2
OP_N, OP_T, OP_H, OP_C = 0, 1, 2, 3
MASK_REAL, MASK_COMPLEX = 0, 1
MASK_CONJ, MASK_ONE_MINUS, MASK_REAL_OUT, MASK_ACCUMULATE = 1, 2, 4, 8
ROUTE_AXIS_REG, ROUTE_AXIS_GENERIC, ROUTE_FOCUS_V2 = 1, 2, 4
# route 3 counted a second focus pair, since removed: the code is retired (no launch counts on it, so its counter reads 0),
# and the name stays so that code written against it keeps working
ROUTE_FOCUS_V1 = 3
ROUTE_MDFT_TC, ROUTE_MDFT_REDUCE, ROUTE_CGEMM = 5, 6, 7
ROUTE_CENTROID, ROUTE_PSI = 8, 9


def route_code(kind, L=0, flags=0):
    """the `route` argument of pb_route_launch_count: the 32-bit int the C side forms (kinds 8 and up are negative)"""
    code = (kind << 28 | L << 8 | flags) & 0xFFFFFFFF
    return code - (1 << 32) if code >> 31 else code

_vp, _i, _ll, _d = C.c_void_p, C.c_int, C.c_longlong, C.c_double

# name -> (restype, argtypes); must list every symbol of include/prysm_b200.h
SIGNATURES = {
    'pb_create': (_i, [C.POINTER(_vp), _i]),
    'pb_destroy': (_i, [_vp]),
    'pb_last_error': (C.c_char_p, [_vp]),
    'pb_version': (C.c_char_p, []),
    'pb_launch_count': (_ll, [_vp]),
    'pb_route_launch_count': (_ll, [_vp, _i]),
    'pb_fft2': (_i, [_vp, _i, _vp, _i, _vp, _i, _d, _i, _i, _ll, _i, _i, _i, _d, _i, _i,
                     _vp, _i, _d, _i, _i, _ll, _vp]),
    'pb_fft2_batch': (_i, [_vp, _i, _vp, _i, _vp, _i, _d, _i, _ll, _ll, _i, _i, _ll, _i, _i, _i, _d, _i, _i,
                           _vp, _i, _d, _i, _i, _ll, _ll, _vp]),
    'pb_fft1': (_i, [_vp, _i, _vp, _i, _i, _ll, _i, _i, _i, _d, _vp, _ll, _vp]),
    'pb_axis_dft': (_i, [_vp, _i, _vp, _i, _i, _ll, _i, _i, _i, _d, _vp, _i, _vp, _i, _vp, _i, _vp, _i, _i, _i, _vp, _ll, _vp]),
    'pb_czt_plan': (_i, [_vp, _i, _i, _i, _i, _d, _d, _i, _d, _d, _d, _vp, _vp, _vp, _vp, _vp]),
    'pb_czt_axis': (_i, [_vp, _i, _vp, _i, _i, _ll, _i, _i, _vp, _i, _vp, _vp, _i, _i, _i, _d, _vp, _ll, _vp]),
    'pb_czt_axis_intensity': (_i, [_vp, _i, _vp, _i, _i, _ll, _i, _i, _vp, _i, _vp, _vp, _i, _i, _i, _d, _i, _d, _vp, _ll, _vp]),
    'pb_polychromatic_czt_work_bytes': (_ll, [_i, _i, _i, _i]),
    'pb_polychromatic_czt': (_i, [_vp, _i, _vp, _i, _vp, _i, _i, _i, _i, C.POINTER(_d), _vp, _vp, _vp]),
    'pb_angular_spectrum': (_i, [_vp, _i, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _i, _vp, _i, _i, _vp]),
    'pb_angular_spectrum_screen': (_i, [_vp, _i, _vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _i, _vp, _i, _i, _vp]),
    'pb_angular_spectrum_vectors': (_i, [_vp, _i, _i, _i, _d, _d, _d, _vp, _vp, _vp]),
    'pb_mdft_basis': (_i, [_vp, _i, C.POINTER(_d), _i, C.POINTER(_d), _i, _i, _vp, _vp]),
    'pb_cgemm': (_i, [_vp, _i, _i, _i, _i, _i, _i, _d, _vp, _ll, _vp, _ll, _vp, _ll, _vp]),
    'pb_mdft_apply': (_i, [_vp, _i, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _d, _i, _i, _vp, _vp]),
    'pb_mdft_work_elems': (_ll, [_i, _i, _i, _i, _i, _i]),
    'pb_mdft_tc_supported': (_i, [_i, _i, _i, _i]),
    'pb_mdft_tc_expand': (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp]),
    'pb_mdft_tc_work_bytes': (_ll, [_i, _i, _i, _i]),
    'pb_mdft_tc_apply': (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _d, _vp, _vp]),
    'pb_phase_screen': (_i, [_vp, _i, _vp, _i, _vp, _d, _ll, _vp, _vp]),
    'pb_intensity': (_i, [_vp, _i, _vp, _ll, _d, _i, _vp, _vp]),
    'pb_binary': (_i, [_vp, _i, _i, _vp, _vp, _d, _d, _i, _ll, _vp, _vp]),
    'pb_mul_outer': (_i, [_vp, _i, _vp, _ll, _i, _i, _vp, _i, _vp, _i, _d, _vp, _ll, _vp]),
    'pb_weighted_sum': (_i, [_vp, _i, _vp, _i, _ll, C.POINTER(_d), _vp, _vp]),
    'pb_otf_normalize': (_i, [_vp, _i, _vp, _i, _i, _i, _vp, _vp, _vp, _vp]),
    'pb_encircled_energy': (_i, [_vp, _i, _vp, _i, _i, _d, C.POINTER(_d), _i, C.POINTER(_d), _vp]),
    'pb_moments': (_i, [_vp, _i, _vp, _i, _i, C.POINTER(_d), _vp]),
    'pb_mask_multiply': (_i, [_vp, _i, _vp, _vp, _vp, _i, _i, _vp, _d, _ll, _vp, _vp]),
    'pb_field_adjoint': (_i, [_vp, _i, _i, _vp, _vp, _vp, _d, _ll, _vp, _vp]),
    'pb_component': (_i, [_vp, _i, _i, _vp, _ll, _vp, _vp]),
    'pb_dot': (_i, [_vp, _i, _vp, _vp, _vp, _ll, C.POINTER(_d), _vp]),
    'pb_mode_projection': (_i, [_vp, _i, _vp, _i, _ll, _vp, _i, C.POINTER(_d), _vp]),
    'pb_otf_adjoint_seed': (_i, [_vp, _i, _i, _vp, _vp, _i, _i, _vp, _vp]),
    'pb_encircled_energy_adjoint_seed': (_i, [_vp, _i, _i, _i, _d, C.POINTER(_d), C.POINTER(_d), _i, _vp, _vp]),
    'pb_vortex_phase': (_i, [_vp, _i, _i, _vp, _vp, _ll, _vp, _vp]),
    'pb_xy_grid': (_i, [_vp, _i, _i, _i, _d, _vp, _vp, _vp, _vp, _vp]),
    'pb_cart_to_polar': (_i, [_vp, _i, _vp, _vp, _ll, _vp, _vp, _vp]),
    'pb_circle': (_i, [_vp, _i, _vp, _ll, _d, _d, _vp, _vp]),
    'pb_jacobi_seq': (_i, [_vp, _i, _vp, _ll, _i, _d, _d, C.POINTER(_i), _vp, _vp]),
    'pb_zernike_seq': (_i, [_vp, _i, _i, _vp, _vp, _ll, _i, C.POINTER(_i), C.POINTER(_i), _i, _vp, _vp]),
    'pb_zernike_sum': (_i, [_vp, _i, _i, _vp, _vp, _ll, _i, C.POINTER(_i), C.POINTER(_i), C.POINTER(_d), _i, _vp, _vp]),
    'pb_balance_scale': (_i, [_vp, _i, _vp, _vp, _ll, _vp, _vp]),
    'pb_pack_complex': (_i, [_vp, _i, _vp, _vp, _vp, _ll, _vp, _vp]),
    'pb_packed_spectrum_product': (_i, [_vp, _i, _vp, _i, _i, _d, _vp, _vp, _vp]),
    'pb_resample_bilinear': (_i, [_vp, _i, _vp, _i, _i, _vp, _vp, _ll, _d, _d, _d, _vp, _d, _d, _vp, _vp]),
    'pb_bindown': (_i, [_vp, _i, _vp, _i, _i, _i, _i, _i, _vp, _vp]),
    'pb_tile': (_i, [_vp, _i, _vp, _i, _i, _i, _i, _d, _vp, _vp]),
    'pb_separable_tf': (_i, [_vp, _i, _i, _vp, _vp, _i, _i, _d, _d, _vp, _vp]),
    'pb_radial_window': (_i, [_vp, _i, _i, _i, _d, _d, _d, _d, _d, _d, _vp, _vp, _vp, _vp]),
    'pb_spline_prefilter': (_i, [_vp, _i, _vp, _i, _i, _i, _vp, _vp]),
    'pb_warp': (_i, [_vp, _i, _vp, _i, _i, _i, _vp, _vp, _i, C.POINTER(_d), _i, _i, _d, _vp, _vp]),
    'pb_dm_scatter': (_i, [_vp, _i, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    'pb_dm_gather': (_i, [_vp, _i, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    'pb_sdf': (_i, [_vp, _i, _i, _vp, _vp, _i, _i, _i, C.POINTER(_d), _i, C.POINTER(_d), _i, _i, _vp, _vp]),
    'pb_sdf_combine': (_i, [_vp, _i, _i, _vp, _vp, _ll, _vp, _vp]),
    'pb_hex_segments': (_i, [_vp, _i, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _i, _d, _vp, _vp, _vp, _vp, _vp]),
    'pb_segment_compose': (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _i, _vp, _ll, _i, _vp, _vp]),
    'pb_segment_compose_adjoint': (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _i, _vp, _i, _vp, _vp, _vp]),
    'pb_jones_planar': (_i, [_vp, _i, _vp, _i, _ll, _ll, _ll, _ll, _ll, _ll, _vp, _vp]),
    'pb_jones_product': (_i, [_vp, _i, _i, _ll, _i, _vp, _i, _i, _vp, _i, C.POINTER(_d), _vp, _vp]),
    'pb_jones_elements': (_i, [_vp, _i, _i, _ll, _vp, _i, C.POINTER(_d), _i, _vp, _vp]),
    'pb_jones_reduce': (_i, [_vp, _i, _i, _ll, _vp, _vp, _vp, _vp]),
    'pb_lp_modes': (_i, [_vp, _i, _vp, _vp, _ll, _d, _i, C.POINTER(_d), _vp, _vp]),
    'pb_overlap': (_i, [_vp, _i, _vp, _ll, _i, _vp, C.POINTER(_vp), _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    'pb_wfs_combine': (_i, [_vp, _i, _ll, _vp, _vp, C.POINTER(_d), _vp, _vp, _i, _vp, _vp]),
    'pb_grating': (_i, [_vp, _i, _i, _ll, _vp, _d, C.POINTER(_d), _i, _vp, _vp, _vp]),
    'pb_psi': (_i, [_vp, _i, _i, C.POINTER(_vp), _vp, _ll, _ll, C.POINTER(_d), C.POINTER(_d), _i, _vp, _vp, _i, _vp,
                    _vp]),
    'pb_expose': (_i, [_vp, _i, _vp, _ll, _ll, _vp, _ll, _ll, _vp, _ll, _ll, C.POINTER(_d), _i, _ll, _i, _vp,
                       _ll, _i, _vp, _vp, _vp]),
    'pb_apply_lut': (_i, [_vp, _i, _vp, _ll, _vp, _ll, _i, _i, _vp, _vp, _vp]),
    'pb_pixel': (_i, [_vp, _i, _vp, _ll, _ll, _vp, _ll, _ll, _ll, _ll, _d, _d, _vp, _vp]),
    'pb_bayer_interleave': (_i, [_vp, _i, C.POINTER(_vp), C.POINTER(_ll), _i, _ll, _ll, _vp, _ll, _vp]),
    'pb_demosaic_deinterlace': (_i, [_vp, _i, _vp, _ll, _ll, _ll, _i, _i, _vp, _vp]),
    'pb_white_balance': (_i, [_vp, _i, _vp, _ll, _ll, _i, C.POINTER(_d), C.POINTER(_d), _vp, _vp]),
    'pb_demosaic_malvar': (_i, [_vp, _i, _vp, _ll, _ll, _ll, _i, _i, _vp, _vp]),
    'pb_bayer_assemble': (_i, [_vp, _i, _vp, _vp, _vp, _vp, _ll, _vp, _vp]),
    'pb_lenslet_screen': (_i, [_vp, _i, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _i, C.POINTER(_d), _d, _d, _vp, _vp]),
    'pb_subaperture_centroids': (_i, [_vp, _i, _vp, _i, _i, _i, _ll, _i, _i, _vp, _vp, _d, _d, _i, _vp, _vp, _vp]),
    'pb_sh_reconstruct': (_i, [_vp, _i, _vp, _i, _ll, _vp, _vp, _vp, _i, _i, _vp, _vp]),
    'pb_qpoly_seq': (_i, [_vp, _i, _i, _i, _vp, _vp, _ll, _i, C.POINTER(_i), C.POINTER(_i), _vp, _vp, _vp]),
    'pb_qpoly_sum': (_i, [_vp, _i, _i, _vp, _vp, _ll, _i, C.POINTER(_i), C.POINTER(_i), C.POINTER(_d), _vp, _vp, _vp,
                          _vp]),
    'pb_qpoly_tables': (_i, [_i, _i, _i, C.POINTER(_d)]),
    'pb_poly_seq': (_i, [_vp, _i, _i, _i, _d, _d, _vp, _ll, _i, C.POINTER(_i), _vp, _vp]),
    'pb_jacobi_radial_sum': (_i, [_vp, _i, _d, _d, _vp, _vp, _ll, _i, C.POINTER(_i), C.POINTER(_d), _d, _vp, _vp, _vp,
                                  _vp]),
    'pb_jacobi_clenshaw': (_i, [_vp, _i, _d, _d, _vp, _ll, _i, C.POINTER(_d), _i, _i, _vp, _vp]),
    'pb_zernike_der': (_i, [_vp, _i, _i, _vp, _vp, _ll, _i, C.POINTER(_i), C.POINTER(_i), _i, _vp, _vp]),
    'pb_zernike_sum_der_xy': (_i, [_vp, _i, _vp, _vp, _ll, _i, C.POINTER(_i), C.POINTER(_i), C.POINTER(_d), _i, _vp,
                                   _vp]),
    'pb_xy_seq': (_i, [_vp, _i, _vp, _vp, _ll, _ll, _i, _i, C.POINTER(_i), C.POINTER(_i), C.POINTER(_i), _vp, _vp]),
    'pb_tensor_sum': (_i, [_vp, _i, _i, _vp, _vp, _ll, _ll, _i, _i, C.POINTER(_i), C.POINTER(_i), C.POINTER(_d), _d, _d,
                           _vp, _vp, _vp, _vp]),
    'pb_stack_eval': (_i, [_vp, _i, _i, _i, _i, _i, _i, C.POINTER(_ll), C.POINTER(_ll), C.POINTER(_vp), _d,
                           C.POINTER(_vp), _vp]),
    'pb_stack_grad': (_i, [_vp, _i, _i, _i, _i, _i, C.POINTER(_ll), C.POINTER(_ll), C.POINTER(_vp), _vp, _vp,
                           C.POINTER(_vp), _vp, _vp]),
    'pb_field_at_depth': (_i, [_vp, _i, _i, _i, _vp, _ll, _vp, _vp, _d, _d, _d, _d, _vp, _vp, _vp, _vp, _vp]),
    'pb_interp2d_linear': (_i, [_vp, _i, _vp, _i, _i, _ll, _vp, _vp, _i, _vp, _vp, _ll, _d, _d, _vp, _vp]),
    'pb_azimuthal_stats': (_i, [_vp, _i, _vp, _i, _i, _vp, _vp, _d, _i, _vp, _vp]),
    'pb_polar_crossings': (_i, [_vp, _i, _vp, _i, _i, _vp, _vp, _d, _d, _i, _i, C.POINTER(_d), _vp]),
    'pb_analytic_radial': (_i, [_vp, _i, _i, _i, _vp, _ll, _d, _d, _vp, _vp]),
}

SDF_POLYGON, SDF_SPIDER, SDF_RECTANGLE, SDF_FILLET_RECTANGLE, SDF_ANNULUS, SDF_OFFSET_CIRCLE = range(6)
SDF_UNION, SDF_INTERSECT, SDF_SUBTRACT = range(3)
SEGMENT_FIELDS, SEGMENT_TILE_Y, SEGMENT_TILE_X, SEGMENT_CHUNK = 6, 32, 64, 2048
JONES_CONST, JONES_PLANES, JONES_SCALAR, JONES_SCALAR_REAL = range(4)
JONES_MATMUL, JONES_HADAMARD = range(2)
JONES_OP_N, JONES_OP_H = range(2)
JONES_FILL, JONES_ROTATION, JONES_RETARDER, JONES_DIATTENUATOR, JONES_VVR = range(5)
JONES_MUELLER, JONES_KRON, JONES_PAULI = range(3)
OVERLAP_CHUNK = 4096
LP_RULE_LP, LP_RULE_SMF = range(2)
LP_NONE, LP_COS, LP_SIN = range(3)
GRATING_SIN_AMP, GRATING_RECTANGLE = range(2)
WB_MAX_BLOCKS = 1024
LENSLET_RECT, LENSLET_RECT_SWAP, LENSLET_RECT_ROTATED, LENSLET_CIRCLE = range(4)
QPOLY_BFS, QPOLY_CON, QPOLY_2D = range(3)
QPOLY_VALUE, QPOLY_DER, QPOLY_DER_XY = range(3)
QPOLY_NMAX = 64
(POLY_JACOBI, POLY_CHEBY1, POLY_CHEBY2, POLY_CHEBY3, POLY_CHEBY4, POLY_LEGENDRE, POLY_HERMITE_HE, POLY_HERMITE_H,
 POLY_LAGUERRE, POLY_DICKSON1, POLY_DICKSON2) = range(11)
POLY_VALUE, POLY_DER, POLY_VALUE_DER = range(3)
POLY_NMAX = 120
CLENSHAW_JMAX = 8
TSUM_MONOMIAL, TSUM_CHEBY1 = range(2)
TF_THINFILM, TF_COATINGS = range(2)
TF_POL_S, TF_POL_P = range(2)
TF_IN_WVL, TF_IN_THETA, TF_IN_N0, TF_IN_NSUB, TF_IN_N, TF_IN_D, TF_NOPS = range(7)
(TF_OUT_R, TF_OUT_T, TF_OUT_E, TF_OUT_H, TF_OUT_REFL, TF_OUT_TRANS, TF_OUT_ABS, TF_OUT_ESQ, TF_OUT_ETA0, TF_OUT_ETASUB,
 TF_NOUT) = range(11)
TF_GRAD_THICKNESS, TF_GRAD_INDEX = 1, 2
TF_DIMS = 4
INTERP_POINTS, INTERP_POLAR = range(2)
AZ_COUNT, AZ_MEAN, AZ_VAR, AZ_MIN, AZ_MAX, AZ_MEDIAN = 1, 2, 4, 8, 16, 32
AZ_ALL = 63
AZ_MAX_NY = 28672
AR_AIRYDISK, AR_AIRYDISK_EFIELD, AR_AIRYDISK_FT, AR_DIFFLIM_MTF, AR_DIFFLIM_NORMALIZED, AR_EE_CIRCULAR = range(6)


def load_library(path=LIB_PATH):
    if not os.path.exists(path):
        raise ImportError(
            f'{path} is missing: build it with `python prysm_b200/build.py` '
            '(prysm_b200 has no CPU fallback)')
    lib = C.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so and the header diverge
        fn.restype = res
        fn.argtypes = args
    return lib


lib = load_library()


class B200Error(RuntimeError):
    """A libprysm_b200 call failed (CUDA error, unsupported shape, bad argument)."""


class Handle:
    """One engine handle per CUDA device (twiddle tables + scratch live here)."""

    def __init__(self, device):
        self._h = _vp()
        rc = lib.pb_create(C.byref(self._h), int(device))
        if rc != 0:
            raise B200Error(f'pb_create(device={device}) failed with status {rc}: is a CUDA device visible?')
        self.device = int(device)

    def check(self, rc):
        if rc != 0:
            msg = lib.pb_last_error(self._h).decode()
            if rc == -1:
                raise ValueError(msg)
            raise B200Error(f'status {rc}: {msg}')

    @property
    def ptr(self):
        return self._h

    def launch_count(self):
        return int(lib.pb_launch_count(self._h))

    def route_launch_count(self, route):
        """kernels launched on one route of the transform kernels (pb_route_launch_count)"""
        return int(lib.pb_route_launch_count(self._h, int(route)))

    def close(self):
        if self._h:
            lib.pb_destroy(self._h)
            self._h = _vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_handles = {}          # (device, raw stream pointer) -> Handle, in least-recently-used order
_pinned = set()        # keys whose handle must outlive the cache (a captured CUDA graph replays into its scratch)
MAX_HANDLES_PER_DEVICE = 8


def handle_for(device_index, stream=0):
    """One handle per (device, stream): a handle's scratch arenas are only ordered by the stream its calls run
    on, so work issued on different streams must not share one (include/prysm_b200.h: 'not thread-safe').
    The cache is bounded: beyond MAX_HANDLES_PER_DEVICE the least recently used un-pinned handle of that device is
    destroyed (pb_destroy synchronises the device first), so short-lived side streams do not accumulate twiddle
    tables and scratch arenas that torch's allocator cannot see."""
    key = (device_index, stream)
    h = _handles.pop(key, None)
    if h is None:
        mine = [k for k in _handles if k[0] == device_index and k not in _pinned]
        while len(mine) >= MAX_HANDLES_PER_DEVICE:
            _handles.pop(mine.pop(0)).close()
        h = Handle(device_index)
    _handles[key] = h          # (re)insert as most recently used
    return h


def pin_handle(device_index, stream):
    """Keep the handle of (device, stream) alive for the life of the process (graphs.capture)."""
    _pinned.add((device_index, stream))


def release_handle(device_index, stream):
    """Destroy the handle of (device, stream) now (explicit close of a side stream's engine state)."""
    _pinned.discard((device_index, stream))
    h = _handles.pop((device_index, stream), None)
    if h is not None:
        h.close()


def launch_count(device_index):
    """Kernels launched on `device_index` through any stream's handle."""
    return sum(h.launch_count() for (d, _), h in _handles.items() if d == device_index)


def version():
    return lib.pb_version().decode()
