"""ctypes binding of liboctfusion_b200.so (the C ABI declared in include/octfusion_b200.h).

There is NO CPU fallback: if the library cannot be loaded every operator raises.  The library
is built in-tree by `octfusion_b200.build` (nvcc, sm_90a); when the .so is missing and nvcc is
available it is built on first import, otherwise the import fails loudly.
"""
from __future__ import annotations
import ctypes as C
import os
import torch

from . import build as _build

OF_F32, OF_BF16 = 0, 1
_i32, _i64, _vp, _f32 = C.c_int32, C.c_int64, C.c_void_p, C.c_float


class GemmArgs(C.Structure):
    """struct of_gemm_args (include/octfusion_b200.h) -- field order and types must match."""
    _fields_ = [
        ('a0', _vp), ('lda0', _i64), ('c0', _i32),
        ('a1', _vp), ('lda1', _i64), ('c1', _i32),
        ('tap_tab', _vp), ('tap_extra', _vp),
        ('in_rows', _vp),
        ('taps', _i32),
        ('node_type', _vp), ('ntype', _i32),
        ('w', _vp),
        ('bias', _vp),
        ('row_add', _vp), ('ld_row_add', _i64), ('row_add_idx', _vp),
        ('resid', _vp), ('ld_resid', _i64),
        ('out_rows', _vp),
        ('out', _vp), ('ldo', _i64),
        ('out_f32', _i32),
        ('M', _i32), ('N', _i32),
        ('dtype', _i32),
        ('a_multi', _vp), ('ld_multi', _i64),
        ('nt_block', _vp),
        ('reverse', _i32),
        ('stat_out', _vp), ('stat_chunk_seg', _vp), ('stat_seg_slot', _vp), ('stat_sample', _vp),
        ('stat_rows_per_sample', _i32),
    ]


class OctreeLevels(C.Structure):
    """struct of_octree_levels."""
    _fields_ = [
        ('keys', _vp * 16), ('children', _vp * 16), ('leaf_rank', _vp * 16),
        ('nnum', _i32 * 16),
        ('full_depth', _i32), ('depth', _i32), ('batch', _i32),
    ]


_PROTOS = {
    'of_last_error': (C.c_char_p, []),
    'of_version': (C.c_int, []),
    'of_num_sms': (C.c_int, []),
    'of_launch_count': (C.c_ulonglong, []),
    'of_abi_sizeof_gemm_args': (C.c_int, []),
    'of_abi_sizeof_octree_levels': (C.c_int, []),
    'of_gather_gemm_simt': (C.c_int, [C.POINTER(GemmArgs), _vp]),
    'of_gather_gemm_tc': (C.c_int, [C.POINTER(GemmArgs), _vp]),
    'of_pack_weight_tc_bytes': (_i64, [_i32, _i32, _i32, _i32]),
    'of_pack_weight_tc': (C.c_int, [_vp, _i32, _i32, _i32, _i32, _vp, _vp]),
    'of_repack_weight': (C.c_int, [_vp, _i64, _i64, _i64, _i32, _i32, _i32, _vp, _vp]),
    'of_gn_stats': (C.c_int, [_vp, _i64, _i32, _vp, _i64, _i32, _vp, _vp, _vp, _i32, _i64, _i32, _i32, _vp, _vp]),
    'of_gn_finalize': (C.c_int, [_vp, _i32, _i32, _vp, _i32, _i32, _vp, _i32, _vp, _i32, _vp, _vp, _i32, _i32, _f32, _f32,
                                 _vp, _vp, _vp, _vp, _vp]),
    'of_gn_apply': (C.c_int, [_vp, _i64, _i32, _vp, _i64, _i32, _vp, _i32, _i64, _vp, _vp, _i32, _i32, _vp, _i64, _i32, _vp]),
    'of_attention': (C.c_int, [_vp, _i64, _vp, _i64, _i32, _i32, _i32, _i32, _i32, _vp]),
    'of_linear_small': (C.c_int, [_vp, _i64, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _i64, _vp]),
    'of_timestep_embedding': (C.c_int, [_vp, _i32, _i32, _f32, _vp, _vp]),
    'of_learned_sinusoidal': (C.c_int, [_vp, _vp, _i32, _i32, _vp, _vp]),
    'of_embedding_add': (C.c_int, [_vp, _vp, _i32, _i32, _vp, _vp]),
    'of_ddim_eps_update': (C.c_int, [_vp, _vp, _vp, _vp, _i64, _vp, _i32, _vp]),
    'of_ddpm_x0_update': (C.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _i32, _vp]),
    'of_copy_rows': (C.c_int, [_vp, _i64, _i32, _vp, _vp, _i64, _i32, _vp, _i64, _i32, _vp]),
    'of_scan_scratch_bytes': (_i64, [_i64]),
    'of_leaf_rank': (C.c_int, [_vp, _i32, _vp, _vp, _vp, _vp]),
    'of_exclusive_scan_i32': (C.c_int, [_vp, _vp, _i64, _vp, _vp, _vp]),
    'of_compact_idx': (C.c_int, [_vp, _vp, _i32, _vp, _vp, _vp]),
    'of_graph_rows': (_i64, [C.POINTER(OctreeLevels), _i32]),
    'of_graph_count': (C.c_int, [C.POINTER(OctreeLevels), _i32, _vp, _vp, _vp]),
    'of_graph_fill': (C.c_int, [C.POINTER(OctreeLevels), _i32, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp]),
    'of_histogram_i32': (C.c_int, [_vp, _i64, _i32, _vp, _vp]),
    'of_graph_type_block': (C.c_int, [_vp, _vp, _vp, _i64, _i32, _i32, _vp, _vp]),
    'of_gather_mean_rows': (C.c_int, [_vp, _i64, _i32, _vp, _i64, _i32, _vp, _i32, _i32, _vp, _i64, _vp]),
    'of_graph_edge_count': (C.c_int, [_vp, _vp, _i64, _vp, _vp]),
    'of_graph_edges': (C.c_int, [_vp, _vp, _i64, _i32, _vp, _vp, _vp, _vp, _vp]),
    'of_dense_tap_table': (C.c_int, [_i32, _i32, _i32, _vp, _vp]),
    'of_octree_neigh27': (C.c_int, [C.POINTER(OctreeLevels), _i32, _vp, _vp]),
    'of_mpu_eval': (C.c_int, [C.POINTER(OctreeLevels), _i32, _vp, _i64, _vp, _vp, _vp, _vp]),
    'of_mpu_eval_grid': (C.c_int, [C.POINTER(OctreeLevels), _i32, _i32, _i32, _f32, _f32, _i64, _i64, _vp, _vp, _vp]),
    'of_nn_distance': (C.c_int, [_vp, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp]),
    'of_chamfer_pairwise': (C.c_int, [_vp, _i32, _i32, _vp, _i32, _i32, _vp, _vp]),
    'of_match_cost': (C.c_int, [_vp, _vp, _i32, _i32, _vp, _vp, _vp]),
    'of_emd_cd_pairwise': (C.c_int, [_vp, _i32, _vp, _i32, _i32, _vp, _vp, _vp]),
    'of_emd_exact': (C.c_int, [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp]),
    'of_emd_exact_pairwise': (C.c_int, [_vp, _i32, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp]),
    'of_mc_count': (C.c_int, [_vp, _i32, _f32, _vp, _vp, _vp]),
    'of_mc_emit': (C.c_int, [_vp, _i32, _f32, _vp, _vp, _vp, _vp, _vp]),
    'of_mesh_bbox': (C.c_int, [_vp, _vp, _i32, _vp, _vp]),
    'of_surface_sample': (C.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, C.c_uint64, _vp, _vp, _vp, _vp]),
    'of_octree_build_bytes': (_i64, [_i64, _i32, _i32, _i32]),
    'of_octree_build_levels': (C.c_int, [_vp, _vp, _i64, _i32, _i32, _i32, _vp, _vp, _vp]),
    'of_octree_build_fill': (C.c_int, [_vp, _i64, _i32, _i32, _i32, _i32, _i64, _vp, _vp, _vp]),
    'of_octree_build_signal': (C.c_int, [_vp, _i64, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp]),
    'of_input_feature_nd': (C.c_int, [_vp, _vp, _vp, _i64, _i64, _i32, _vp, _i64, _vp]),
    'of_mesh_components_bytes': (_i64, [_i64, _i64]),
    'of_mesh_components': (C.c_int, [_vp, _i32, _vp, _i32, _vp, _vp, _vp, _vp]),
    'of_mesh_largest_component': (C.c_int, [_vp, _i32, _vp, _i32, _vp, _vp, _vp, _vp, _vp]),
    'of_mesh_compact': (C.c_int, [_vp, _i32, _vp, _i32, _vp, _i32, _vp, _vp, _vp, _vp, _vp]),
}

EMD_MAX_POINTS = 4096              # OF_EMD_MAX_POINTS
CD_PAIRWISE_MAX_POINTS = 49152     # OF_CD_PAIRWISE_MAX_POINTS
MC_MAX_SIZE = 512                  # OF_MC_MAX_SIZE

EXPORTED_SYMBOLS = tuple(_PROTOS)


class LibraryMissing(ImportError):
    pass


ABI_VERSION = 7          # of_version() of the header this binding mirrors


def _load():
    path = _build.LIB
    # (re)build when the library is missing or older than a source / the header -- only where nvcc exists (the GPU
    # box receives the prebuilt .so with the snapshot and has the same sources, so needs_build() is False there)
    if _build.needs_build() and (not os.path.exists(path) or _build.have_nvcc()):
        try:
            _build.build()
        except Exception as e:  # noqa: BLE001
            if not os.path.exists(path):
                raise LibraryMissing(
                    'octfusion_b200: CUDA library %s is missing and could not be built (%s). '
                    'There is no CPU fallback; run `python -m octfusion_b200.build`.' % (path, e)) from e
            raise
    lib = C.CDLL(path)
    for name, (res, args) in _PROTOS.items():
        fn = getattr(lib, name)          # AttributeError here = header / library mismatch
        fn.restype = res
        fn.argtypes = args
    # a stale library with another struct layout would read garbage pointers: refuse it
    got = (lib.of_version(), lib.of_abi_sizeof_gemm_args(), lib.of_abi_sizeof_octree_levels())
    want = (ABI_VERSION, C.sizeof(GemmArgs), C.sizeof(OctreeLevels))
    if got != want:
        raise LibraryMissing('octfusion_b200: %s has ABI (version, sizeof gemm_args, sizeof octree_levels) = %s, this '
                             'binding expects %s -- rebuild with `python -m octfusion_b200.build --force`' % (path, got, want))
    return lib


lib = _load()


def last_error() -> str:
    return lib.of_last_error().decode('utf-8', 'replace')


def check(rc: int, what: str = ''):
    if rc != 0:
        raise RuntimeError('octfusion_b200 %s failed (rc=%d): %s' % (what, rc, last_error()))


def ptr(t):
    """device pointer of a tensor (or None)."""
    if t is None:
        return None
    return C.c_void_p(t.data_ptr())


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def dt(t) -> int:
    if t.dtype == torch.float32:
        return OF_F32
    if t.dtype == torch.bfloat16:
        return OF_BF16
    raise TypeError('octfusion_b200: unsupported activation dtype %s (float32 or bfloat16)' % t.dtype)


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError('octfusion_b200: tensors must live on a CUDA device -- there is no CPU path')


def launch_count() -> int:
    return int(lib.of_launch_count())
