"""ctypes mirror of the reference's safe-ish Rust wrappers (lib/kvbm-kernels/src/tensor_kernels.rs).

Same function names, argument meaning and error behaviour as the Rust crate:
  vectorized_copy      tensor_kernels.rs:232-250   -> kvbm_kernels_launch_vectorized_copy
  memcpy_batch         tensor_kernels.rs:139-175   -> kvbm_kernels_memcpy_batch
  universal_from_block tensor_kernels.rs:177-215   -> kvbm_kernels_launch_universal_from_block
  block_from_universal tensor_kernels.rs:217-...   -> kvbm_kernels_launch_block_from_universal
  is_memcpy_batch_available / is_using_stubs       tensor_kernels.rs:111-137
plus the v2 paged entry point (include/kvbm_kernels.h part 2).  Every function returns the raw
cudaError_t (0 == cudaSuccess) like the FFI does; `check()` turns it into an exception.
"""
from __future__ import annotations

import ctypes as C
import enum
from typing import Optional, Sequence, Tuple

from . import _lib

MAX_DESTINATIONS = 8


class TensorDataType(enum.IntEnum):
    F16 = 0
    BF16 = 1
    F32 = 2
    F64 = 3


class BlockLayout(enum.IntEnum):
    NHD = 0
    HND = 1


class MemcpyBatchMode(enum.IntEnum):
    BatchedWithFallback = 0
    FallbackOnly = 1
    BatchWithoutFallback = 2


class KvBlockLayout(enum.IntEnum):
    """KVBM_KV_* -- lib/kvbm-physical/src/layout/kv_block_layout.rs:40-76 (dimension order of one block, head_dim innermost)"""
    Unknown = 0
    UniversalTP = 1      # [nh, nl, no, nt, hd]
    UniversalPP = 2      # [nl, nh, no, nt, hd]
    OperationalHND = 3   # [nl, no, nh, nt, hd]
    OperationalNHD = 4   # [nl, no, nt, nh, hd]
    Custom = 5


class CastMode(enum.IntEnum):
    NONE = 0
    FP8E4M3_TO_BF16 = 1
    BF16_TO_FP8E4M3 = 2


CUDA_SUCCESS = 0
CUDA_ERROR_INVALID_VALUE = 1


class CudaError(RuntimeError):
    def __init__(self, code: int, what: str):
        super().__init__(f"{what} failed: cudaError_t={code}")
        self.code = code


def check(code: int, what: str = "kvbm_kernels") -> None:
    if code != CUDA_SUCCESS:
        raise CudaError(code, what)


class PagedLayout(C.Structure):
    """struct kvbm_paged_layout"""
    _fields_ = [
        ("layer_base", C.c_void_p),
        ("block_stride", C.c_uint64),
        ("outer_stride", C.c_uint64),
        ("region_bytes", C.c_uint32),
        ("num_layers", C.c_uint32),
        ("outer_dim", C.c_uint32),
        ("num_blocks", C.c_uint32),
    ]


class PagedDst(C.Structure):
    """struct kvbm_paged_dst"""
    _fields_ = [
        ("layout", PagedLayout),
        ("src_block_ids", C.c_void_p),
        ("dst_block_ids", C.c_void_p),
        ("done_flag", C.c_void_p),
        ("layer_done_flags", C.c_void_p),
    ]


class PermuteSide(C.Structure):
    """struct kvbm_permute_side"""
    _fields_ = [("layout", PagedLayout), ("block_ids", C.c_void_p), ("kv_layout", C.c_int)]


class PermuteSource(C.Structure):
    """struct kvbm_permute_source: one source of `paged_permute_gather` (a side, its head count and its head window)"""
    _fields_ = [("side", PermuteSide), ("num_heads", C.c_uint32), ("src_head_begin", C.c_uint32), ("dst_head_begin", C.c_uint32),
                ("head_count", C.c_uint32)]


class StageSource(C.Structure):
    """struct kvbm_stage_source: one source of `paged_stage_gather` (a gather source whose side has the pool's own num_layers,
    and its layer window: source layers [src_layer_begin, +layer_count) land as destination layers [dst_layer_begin, +layer_count))"""
    _fields_ = [("src", PermuteSource), ("src_layer_begin", C.c_uint32), ("dst_layer_begin", C.c_uint32), ("layer_count", C.c_uint32)]


class RepageSeq(C.Structure):
    """struct kvbm_repage_seq: one sequence's token range in a batch (host memory)"""
    _fields_ = [("token_begin", C.c_uint32), ("token_end", C.c_uint32)]


class RepageUnit(C.Structure):
    """struct kvbm_repage_unit: one block of the larger-page side of a batch, 16 B (`repage_batch_units` writes them)"""
    _fields_ = [("q0", C.c_uint32), ("tokens", C.c_uint32), ("small_k", C.c_uint32), ("seq", C.c_uint32)]


class RouteSeq(C.Structure):
    """struct kvbm_route_seq: one sequence of a routed scatter, its token range and its targets (bit t: target t; host memory)"""
    _fields_ = [("token_begin", C.c_uint32), ("token_end", C.c_uint32), ("targets", C.c_uint32)]


class RouteUnit(C.Structure):
    """struct kvbm_route_unit: RepageUnit with the sequence's targets in place of seq, 16 B (`repage_route_units` writes them)"""
    _fields_ = [("q0", C.c_uint32), ("tokens", C.c_uint32), ("small_k", C.c_uint32), ("targets", C.c_uint32)]


class RepageAnypageUnit(C.Structure):
    """struct kvbm_repage_anypage_unit: RepageUnit with the block's phase in place of seq, 16 B (`repage_anypage_units` writes them)"""
    _fields_ = [("q0", C.c_uint32), ("tokens", C.c_uint32), ("small_k", C.c_uint32), ("phase", C.c_uint32)]


class RouteAnypageUnit(C.Structure):
    """struct kvbm_route_anypage_unit: RouteUnit for pages that need not divide, 16 B: route = targets | phase << 16
    (`repage_route_anypage_units` writes them)"""
    _fields_ = [("q0", C.c_uint32), ("tokens", C.c_uint32), ("small_k", C.c_uint32), ("route", C.c_uint32)]


class ScatterTarget(C.Structure):
    """struct kvbm_scatter_target: one target of `paged_repage_scatter` (a destination side, its head count, one head window, one
    layer window and its nullable done flag)"""
    _fields_ = [("side", PermuteSide), ("num_heads", C.c_uint32), ("src_head_begin", C.c_uint32), ("dst_head_begin", C.c_uint32),
                ("head_count", C.c_uint32), ("src_layer_begin", C.c_uint32), ("dst_layer_begin", C.c_uint32), ("layer_count", C.c_uint32),
                ("done_flag", C.c_void_p)]


GATHER_MAX_SOURCES = 16      # KVBM_GATHER_MAX_SOURCES
GATHER_MAX_HEADS = 256       # KVBM_GATHER_MAX_HEADS


class PermuteStream(C.Structure):
    """struct kvbm_permute_stream: the gate of `paged_permute_gather_streamed` / `paged_repage_gather_streamed`"""
    _fields_ = [
        ("layer_ready_flags", C.c_void_p * GATHER_MAX_SOURCES),  # per source (srcs[] index): its [num_layers] ready flags
        ("layer_done_flags", C.c_void_p),
        ("done_flag", C.c_void_p),
        ("epoch", C.c_uint32),
        ("sync_workspace", C.c_void_p),   # u32[sync_workspace_words(num_layers)], zeroed (spinning form)
        ("completion_flag", C.c_void_p),
        ("completion_value", C.c_uint32),
        ("gate_mode", C.c_int),
        ("gate_timeout_ms", C.c_int),
        ("max_ctas", C.c_int),
    ]


class PagedCopyOpts(C.Structure):
    """struct kvbm_paged_copy_opts"""
    _fields_ = [
        ("epoch", C.c_uint32),
        ("layer_ready_flags", C.c_void_p),
        ("sync_workspace", C.c_void_p),
        ("max_ctas", C.c_int),
        ("warps_per_cta", C.c_int),
        ("stages", C.c_int),
        ("tile_bytes", C.c_int),
        ("force_simt", C.c_int),
        ("completion_flag", C.c_void_p),
        ("completion_value", C.c_uint32),
        ("stores_in_flight", C.c_int),
        ("cache_hint", C.c_int),
        ("variant", C.c_int),
        ("gate_timeout_ms", C.c_int),
        ("multicast", C.c_int),
        ("gate_mode", C.c_int),
        ("static_schedule", C.c_int),
        ("cast_scales", C.c_void_p),      # device-accessible float[num_layers * outer_dim]: the fp8 side's scales, or None
    ]


def sync_workspace_words(num_layers: int) -> int:
    """KVBM_SYNC_WORKSPACE_WORDS: u32 words of PagedCopyOpts.sync_workspace (per-layer counters + control words)."""
    return int(num_layers) + 4


_configured = False


def lib() -> C.CDLL:
    global _configured
    L = _lib.load(_lib.KERNELS_SO)
    if not _configured:
        vp, sz, i = C.c_void_p, C.c_size_t, C.c_int
        L.kvbm_kernels_launch_vectorized_copy.argtypes = [vp, vp, sz, i, vp]
        L.kvbm_kernels_launch_vectorized_copy.restype = i
        L.kvbm_kernels_memcpy_batch.argtypes = [vp, vp, sz, sz, i, vp]
        L.kvbm_kernels_memcpy_batch.restype = i
        for f in (L.kvbm_kernels_launch_universal_from_block, L.kvbm_kernels_launch_block_from_universal):
            f.argtypes = [vp, vp, sz, sz, sz, sz, sz, sz, i, i, vp]
            f.restype = i
        L.kvbm_kernels_has_memcpy_batch_async.restype = C.c_bool
        L.kvbm_kernels_is_stub_build.restype = C.c_bool
        L.kvbm_kernels_paged_copy_v2.argtypes = [C.POINTER(PagedLayout), C.POINTER(PagedDst), i, i, i, i, i,
                                                 C.POINTER(PagedCopyOpts), vp]
        L.kvbm_kernels_paged_copy_v2.restype = i
        L.kvbm_kernels_paged_permute.argtypes = [C.POINTER(PermuteSide), C.POINTER(PermuteSide), i, i, i, C.c_uint32, C.c_uint32,
                                                 C.c_uint32, vp, C.c_uint32, vp, C.c_uint32, vp]
        L.kvbm_kernels_paged_permute.restype = i
        L.kvbm_kernels_paged_permute_cast.argtypes = [C.POINTER(PermuteSide), C.POINTER(PermuteSide), i, i, i, C.c_uint32, C.c_uint32,
                                                      C.c_uint32, i, vp, C.c_uint32, vp, C.c_uint32, vp]
        L.kvbm_kernels_paged_permute_cast.restype = i
        L.kvbm_kernels_paged_permute_heads.argtypes = [C.POINTER(PermuteSide), C.POINTER(PermuteSide), i, i, i, C.c_uint32, C.c_uint32,
                                                       C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, i, vp, C.c_uint32, vp,
                                                       C.c_uint32, vp]
        L.kvbm_kernels_paged_permute_heads.restype = i
        L.kvbm_kernels_paged_permute_heads_scaled.argtypes = [C.POINTER(PermuteSide), C.POINTER(PermuteSide), i, i, i, C.c_uint32,
                                                              C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, i, vp,
                                                              vp, C.c_uint32, vp, C.c_uint32, vp]
        L.kvbm_kernels_paged_permute_heads_scaled.restype = i
        L.kvbm_kernels_paged_permute_gather.argtypes = [C.POINTER(PermuteSource), i, C.POINTER(PermuteSide), C.c_uint32, i, i, i, C.c_uint32,
                                                        C.c_uint32, i, vp, C.c_uint32, vp, C.c_uint32, vp]
        L.kvbm_kernels_paged_permute_gather.restype = i
        L.kvbm_kernels_paged_permute_gather_scaled.argtypes = [C.POINTER(PermuteSource), i, C.POINTER(PermuteSide), C.c_uint32, i, i, i,
                                                               C.c_uint32, C.c_uint32, i, vp, vp, C.c_uint32, vp, C.c_uint32, vp]
        L.kvbm_kernels_paged_permute_gather_scaled.restype = i
        L.kvbm_kernels_paged_repage.argtypes = [C.POINTER(PermuteSide), C.c_uint32, C.POINTER(PermuteSide), C.c_uint32, C.c_uint32,
                                                C.c_uint32, i, i, C.c_uint32, C.c_uint32, i, vp, vp, C.c_uint32, vp, C.c_uint32, vp]
        L.kvbm_kernels_paged_repage.restype = i
        L.kvbm_kernels_paged_repage_gather.argtypes = [C.POINTER(PermuteSource), i, C.c_uint32, C.POINTER(PermuteSide), C.c_uint32,
                                                       C.c_uint32, C.c_uint32, C.c_uint32, i, i, C.c_uint32, i, vp, vp, C.c_uint32, vp,
                                                       C.c_uint32, vp]
        L.kvbm_kernels_paged_repage_gather.restype = i
        L.kvbm_kernels_paged_permute_gather_streamed.argtypes = [C.POINTER(PermuteSource), i, C.POINTER(PermuteSide), C.c_uint32, i, i, i,
                                                                 C.c_uint32, C.c_uint32, i, vp, C.POINTER(PermuteStream), vp]
        L.kvbm_kernels_paged_permute_gather_streamed.restype = i
        L.kvbm_kernels_paged_repage_gather_streamed.argtypes = [C.POINTER(PermuteSource), i, C.c_uint32, C.POINTER(PermuteSide), C.c_uint32,
                                                                C.c_uint32, C.c_uint32, C.c_uint32, i, i, C.c_uint32, i, vp,
                                                                C.POINTER(PermuteStream), vp]
        L.kvbm_kernels_paged_repage_gather_streamed.restype = i
        L.kvbm_kernels_paged_stage_gather.argtypes = [C.POINTER(StageSource), i, C.POINTER(PermuteSide), C.c_uint32, i, i, i, C.c_uint32,
                                                      C.c_uint32, i, vp, vp, C.c_uint32, vp, C.c_uint32, vp]
        L.kvbm_kernels_paged_stage_gather.restype = i
        L.kvbm_kernels_paged_stage_gather_streamed.argtypes = [C.POINTER(StageSource), i, C.POINTER(PermuteSide), C.c_uint32, i, i, i,
                                                               C.c_uint32, C.c_uint32, i, vp, C.POINTER(PermuteStream), vp]
        L.kvbm_kernels_paged_stage_gather_streamed.restype = i
        L.kvbm_kernels_paged_stage_repage_gather.argtypes = [C.POINTER(StageSource), i, C.c_uint32, C.POINTER(PermuteSide), C.c_uint32,
                                                             C.c_uint32, C.c_uint32, C.c_uint32, i, i, C.c_uint32, i, vp, vp, C.c_uint32,
                                                             vp, C.c_uint32, vp]
        L.kvbm_kernels_paged_stage_repage_gather.restype = i
        L.kvbm_kernels_paged_stage_repage_gather_streamed.argtypes = [C.POINTER(StageSource), i, C.c_uint32, C.POINTER(PermuteSide),
                                                                      C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, i, i, C.c_uint32, i,
                                                                      vp, C.POINTER(PermuteStream), vp]
        L.kvbm_kernels_paged_stage_repage_gather_streamed.restype = i
        L.kvbm_kernels_repage_batch_units.argtypes = [vp, sz, C.c_uint32, C.c_uint32, vp, sz, C.POINTER(sz), C.POINTER(sz), C.POINTER(sz)]
        L.kvbm_kernels_repage_batch_units.restype = i
        L.kvbm_kernels_paged_stage_repage_gather_batch.argtypes = [C.POINTER(StageSource), i, C.c_uint32, C.POINTER(PermuteSide), C.c_uint32,
                                                                   C.c_uint32, vp, sz, vp, sz, i, i, C.c_uint32, i, vp, vp, C.c_uint32, vp,
                                                                   C.c_uint32, vp]
        L.kvbm_kernels_paged_stage_repage_gather_batch.restype = i
        L.kvbm_kernels_paged_stage_repage_gather_batch_streamed.argtypes = [C.POINTER(StageSource), i, C.c_uint32, C.POINTER(PermuteSide),
                                                                            C.c_uint32, C.c_uint32, vp, sz, vp, sz, i, i, C.c_uint32, i, vp,
                                                                            C.POINTER(PermuteStream), vp]
        L.kvbm_kernels_paged_stage_repage_gather_batch_streamed.restype = i
        L.kvbm_kernels_paged_repage_scatter.argtypes = [C.POINTER(PermuteSide), C.c_uint32, C.c_uint32, C.POINTER(ScatterTarget), i,
                                                        C.c_uint32, C.c_uint32, C.c_uint32, i, i, C.c_uint32, i, vp, C.c_uint32, vp,
                                                        C.c_uint32, vp]
        L.kvbm_kernels_paged_repage_scatter.restype = i
        L.kvbm_kernels_paged_repage_scatter_streamed.argtypes = [C.POINTER(PermuteSide), C.c_uint32, C.c_uint32, C.POINTER(ScatterTarget),
                                                                 i, C.c_uint32, C.c_uint32, C.c_uint32, i, i, C.c_uint32, i, vp,
                                                                 C.POINTER(PermuteStream), vp]
        L.kvbm_kernels_paged_repage_scatter_streamed.restype = i
        L.kvbm_kernels_paged_repage_scatter_batch.argtypes = [C.POINTER(PermuteSide), C.c_uint32, C.c_uint32, C.POINTER(ScatterTarget), i,
                                                              C.c_uint32, vp, sz, vp, sz, i, i, C.c_uint32, i, vp, C.c_uint32, vp, C.c_uint32,
                                                              vp]
        L.kvbm_kernels_paged_repage_scatter_batch.restype = i
        L.kvbm_kernels_paged_repage_scatter_batch_streamed.argtypes = [C.POINTER(PermuteSide), C.c_uint32, C.c_uint32,
                                                                       C.POINTER(ScatterTarget), i, C.c_uint32, vp, sz, vp, sz, i, i,
                                                                       C.c_uint32, i, vp, C.POINTER(PermuteStream), vp]
        L.kvbm_kernels_paged_repage_scatter_batch_streamed.restype = i
        L.kvbm_kernels_repage_route_units.argtypes = [vp, sz, C.c_uint32, C.c_uint32, vp, sz, C.POINTER(sz), C.POINTER(sz), C.POINTER(sz)]
        L.kvbm_kernels_repage_route_units.restype = i
        L.kvbm_kernels_paged_repage_scatter_routed.argtypes = L.kvbm_kernels_paged_repage_scatter_batch.argtypes
        L.kvbm_kernels_paged_repage_scatter_routed.restype = i
        L.kvbm_kernels_paged_repage_scatter_routed_streamed.argtypes = L.kvbm_kernels_paged_repage_scatter_batch_streamed.argtypes
        L.kvbm_kernels_paged_repage_scatter_routed_streamed.restype = i
        L.kvbm_kernels_paged_stage_repage_gather_routed.argtypes = L.kvbm_kernels_paged_stage_repage_gather_batch.argtypes
        L.kvbm_kernels_paged_stage_repage_gather_routed.restype = i
        L.kvbm_kernels_paged_stage_repage_gather_routed_streamed.argtypes = L.kvbm_kernels_paged_stage_repage_gather_batch_streamed.argtypes
        L.kvbm_kernels_paged_stage_repage_gather_routed_streamed.restype = i
        L.kvbm_kernels_repage_anypage_units.argtypes = L.kvbm_kernels_repage_batch_units.argtypes
        L.kvbm_kernels_repage_anypage_units.restype = i
        L.kvbm_kernels_paged_stage_repage_gather_anypage.argtypes = L.kvbm_kernels_paged_stage_repage_gather_batch.argtypes
        L.kvbm_kernels_paged_stage_repage_gather_anypage.restype = i
        L.kvbm_kernels_paged_stage_repage_gather_anypage_streamed.argtypes = L.kvbm_kernels_paged_stage_repage_gather_batch_streamed.argtypes
        L.kvbm_kernels_paged_stage_repage_gather_anypage_streamed.restype = i
        L.kvbm_kernels_paged_repage_scatter_anypage.argtypes = L.kvbm_kernels_paged_repage_scatter_batch.argtypes
        L.kvbm_kernels_paged_repage_scatter_anypage.restype = i
        L.kvbm_kernels_paged_repage_scatter_anypage_streamed.argtypes = L.kvbm_kernels_paged_repage_scatter_batch_streamed.argtypes
        L.kvbm_kernels_paged_repage_scatter_anypage_streamed.restype = i
        L.kvbm_kernels_repage_route_anypage_units.argtypes = L.kvbm_kernels_repage_route_units.argtypes
        L.kvbm_kernels_repage_route_anypage_units.restype = i
        L.kvbm_kernels_paged_repage_scatter_routed_anypage.argtypes = L.kvbm_kernels_paged_repage_scatter_batch.argtypes
        L.kvbm_kernels_paged_repage_scatter_routed_anypage.restype = i
        L.kvbm_kernels_paged_repage_scatter_routed_anypage_streamed.argtypes = L.kvbm_kernels_paged_repage_scatter_batch_streamed.argtypes
        L.kvbm_kernels_paged_repage_scatter_routed_anypage_streamed.restype = i
        L.kvbm_kernels_paged_stage_repage_gather_routed_anypage.argtypes = L.kvbm_kernels_paged_stage_repage_gather_batch.argtypes
        L.kvbm_kernels_paged_stage_repage_gather_routed_anypage.restype = i
        L.kvbm_kernels_paged_stage_repage_gather_routed_anypage_streamed.argtypes = (
            L.kvbm_kernels_paged_stage_repage_gather_batch_streamed.argtypes)
        L.kvbm_kernels_paged_stage_repage_gather_routed_anypage_streamed.restype = i
        L.kvbm_kernels_permute_strides.argtypes = [i, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint64,
                                                   C.POINTER(C.c_uint64)]
        L.kvbm_kernels_permute_strides.restype = i
        L.kvbm_kernels_set_flags.argtypes = [vp, i, i, C.c_uint32, vp]
        L.kvbm_kernels_set_flags.restype = i
        L.kvbm_kernels_wait_flag.argtypes = [vp, C.c_uint32, vp]
        L.kvbm_kernels_wait_flag.restype = i
        L.kvbm_kernels_stream_wait_event.argtypes = [vp, vp]
        L.kvbm_kernels_stream_wait_event.restype = i
        L.kvbm_kernels_launch_count.restype = C.c_uint64
        L.kvbm_kernels_build_info.restype = C.c_char_p
        _configured = True
    return L


EXPORTED_SYMBOLS = [
    "kvbm_kernels_launch_vectorized_copy", "kvbm_kernels_memcpy_batch",
    "kvbm_kernels_launch_universal_from_block", "kvbm_kernels_launch_block_from_universal",
    "kvbm_kernels_has_memcpy_batch_async", "kvbm_kernels_is_stub_build",
    "kvbm_kernels_paged_copy_v2", "kvbm_kernels_set_flags", "kvbm_kernels_wait_flag", "kvbm_kernels_stream_wait_event",
    "kvbm_kernels_launch_count", "kvbm_kernels_build_info", "kvbm_kernels_gate_would_spin", "kvbm_kernels_paged_permute",
    "kvbm_kernels_permute_strides", "kvbm_kernels_paged_permute_cast", "kvbm_kernels_paged_permute_heads",
    "kvbm_kernels_paged_permute_gather", "kvbm_kernels_paged_permute_heads_scaled", "kvbm_kernels_paged_permute_gather_scaled",
    "kvbm_kernels_paged_repage", "kvbm_kernels_paged_repage_gather", "kvbm_kernels_paged_permute_gather_streamed",
    "kvbm_kernels_paged_repage_gather_streamed", "kvbm_kernels_paged_stage_gather", "kvbm_kernels_paged_stage_gather_streamed",
    "kvbm_kernels_paged_stage_repage_gather", "kvbm_kernels_paged_stage_repage_gather_streamed",
    "kvbm_kernels_repage_batch_units", "kvbm_kernels_paged_stage_repage_gather_batch",
    "kvbm_kernels_paged_stage_repage_gather_batch_streamed", "kvbm_kernels_paged_repage_scatter",
    "kvbm_kernels_paged_repage_scatter_streamed", "kvbm_kernels_paged_repage_scatter_batch",
    "kvbm_kernels_paged_repage_scatter_batch_streamed", "kvbm_kernels_repage_route_units", "kvbm_kernels_paged_repage_scatter_routed",
    "kvbm_kernels_paged_repage_scatter_routed_streamed", "kvbm_kernels_paged_stage_repage_gather_routed",
    "kvbm_kernels_paged_stage_repage_gather_routed_streamed", "kvbm_kernels_repage_anypage_units",
    "kvbm_kernels_paged_stage_repage_gather_anypage", "kvbm_kernels_paged_stage_repage_gather_anypage_streamed",
    "kvbm_kernels_paged_repage_scatter_anypage", "kvbm_kernels_paged_repage_scatter_anypage_streamed",
    "kvbm_kernels_repage_route_anypage_units", "kvbm_kernels_paged_repage_scatter_routed_anypage",
    "kvbm_kernels_paged_repage_scatter_routed_anypage_streamed", "kvbm_kernels_paged_stage_repage_gather_routed_anypage",
    "kvbm_kernels_paged_stage_repage_gather_routed_anypage_streamed",
]


def scales_ptr(cast_scales) -> Optional[int]:
    """Address of a cast-scale array: None, an int address, or a contiguous float32 tensor / array (torch: data_ptr(), numpy:
    ctypes.data).  The array must outlive the launch."""
    if cast_scales is None or isinstance(cast_scales, int):
        return cast_scales or None
    if hasattr(cast_scales, "data_ptr"):
        import torch
        if cast_scales.dtype != torch.float32 or not cast_scales.is_contiguous():
            raise ValueError("cast_scales must be a contiguous float32 tensor")
        return cast_scales.data_ptr()
    import numpy as np
    if cast_scales.dtype != np.float32 or not cast_scales.flags["C_CONTIGUOUS"]:
        raise ValueError("cast_scales must be a contiguous float32 array")
    return cast_scales.ctypes.data

GATE_AUTO, GATE_SPIN, GATE_STREAM_WAIT = 0, 1, 2


def gate_would_spin() -> bool:
    """True when gated transfers spin in ONE launch (eager CUDA module loading); False when they gate on the stream."""
    return bool(lib().kvbm_kernels_gate_would_spin())


def is_memcpy_batch_available() -> bool:
    return bool(lib().kvbm_kernels_has_memcpy_batch_async())


def is_using_stubs() -> bool:
    return bool(lib().kvbm_kernels_is_stub_build())


def launch_count() -> int:
    return int(lib().kvbm_kernels_launch_count())


def vectorized_copy(src_ptrs: int, dst_ptrs: int, copy_size_bytes: int, num_pairs: int, stream: int) -> int:
    """src_ptrs/dst_ptrs: address of a DEVICE-ACCESSIBLE table of `num_pairs` pointers."""
    return lib().kvbm_kernels_launch_vectorized_copy(src_ptrs, dst_ptrs, copy_size_bytes, num_pairs, stream)


def memcpy_batch(src_ptrs: Optional[Sequence[int]], dst_ptrs: Optional[Sequence[int]], size_per_copy: int,
                 num_copies: int, mode: MemcpyBatchMode, stream: int) -> int:
    """src_ptrs/dst_ptrs: HOST sequences of addresses (None -> NULL table)."""
    s = (C.c_void_p * len(src_ptrs))(*src_ptrs) if src_ptrs is not None else None
    d = (C.c_void_p * len(dst_ptrs))(*dst_ptrs) if dst_ptrs is not None else None
    return lib().kvbm_kernels_memcpy_batch(s, d, size_per_copy, num_copies, int(mode), stream)


def universal_from_block(universal_ptrs: int, block_ptrs: int, num_blocks: int, nh: int, nl: int, no: int,
                         nt: int, hd: int, dtype: int, layout: int, stream: int) -> int:
    return lib().kvbm_kernels_launch_universal_from_block(universal_ptrs, block_ptrs, num_blocks, nh, nl, no, nt,
                                                          hd, int(dtype), int(layout), stream)


def block_from_universal(universal_ptrs: int, block_ptrs: int, num_blocks: int, nh: int, nl: int, no: int,
                         nt: int, hd: int, dtype: int, layout: int, stream: int) -> int:
    return lib().kvbm_kernels_launch_block_from_universal(universal_ptrs, block_ptrs, num_blocks, nh, nl, no, nt,
                                                          hd, int(dtype), int(layout), stream)


def paged_copy(src: PagedLayout, dsts: Sequence[PagedDst], num_blocks: int, layer_begin: int, layer_end: int,
               cast_mode: int = 0, opts: Optional[PagedCopyOpts] = None, stream: int = 0) -> int:
    arr = (PagedDst * max(1, len(dsts)))(*dsts)
    return lib().kvbm_kernels_paged_copy_v2(C.byref(src), arr, len(dsts), num_blocks, layer_begin, layer_end,
                                            int(cast_mode), C.byref(opts) if opts is not None else None, stream)


def paged_permute(src: PermuteSide, dst: PermuteSide, num_blocks: int, layer_begin: int, layer_end: int, num_heads: int,
                  page_size: int, row_bytes: int, done_flag: int = 0, epoch: int = 0, completion_flag: int = 0,
                  completion_value: int = 0, stream: int = 0) -> int:
    """Blocks src.block_ids[i] -> dst.block_ids[i], every element moved from its place under src.kv_layout to its place under
    dst.kv_layout; row_bytes = head_dim * element size.  include/kvbm_kernels.h (kvbm_kernels_paged_permute)."""
    return lib().kvbm_kernels_paged_permute(C.byref(src), C.byref(dst), num_blocks, layer_begin, layer_end, num_heads, page_size,
                                            row_bytes, done_flag or None, epoch, completion_flag or None, completion_value, stream)


def paged_permute_cast(src: PermuteSide, dst: PermuteSide, num_blocks: int, layer_begin: int, layer_end: int, num_heads: int,
                       page_size: int, src_row_bytes: int, cast_mode: int, done_flag: int = 0, epoch: int = 0, completion_flag: int = 0,
                       completion_value: int = 0, stream: int = 0) -> int:
    """`paged_permute` with the fp8 e4m3 <-> bf16 cast fused in (CastMode); src_row_bytes = head_dim * source element size, the
    destination row is twice / half / equal to it.  include/kvbm_kernels.h (kvbm_kernels_paged_permute_cast)."""
    return lib().kvbm_kernels_paged_permute_cast(C.byref(src), C.byref(dst), num_blocks, layer_begin, layer_end, num_heads, page_size,
                                                 src_row_bytes, int(cast_mode), done_flag or None, epoch, completion_flag or None,
                                                 completion_value, stream)


def paged_permute_heads(src: PermuteSide, dst: PermuteSide, num_blocks: int, layer_begin: int, layer_end: int, src_num_heads: int,
                        src_head_begin: int, dst_num_heads: int, dst_head_begin: int, head_count: int, page_size: int, src_row_bytes: int,
                        cast_mode: int = 0, done_flag: int = 0, epoch: int = 0, completion_flag: int = 0, completion_value: int = 0,
                        stream: int = 0, cast_scales=None) -> int:
    """`paged_permute_cast` over a head window on each side (a TP re-shard): source heads [src_head_begin, +head_count) land as
    destination heads [dst_head_begin, +head_count); each side has its own head count and every destination byte outside the
    window keeps its value.  `cast_scales` (float32[num_layers * outer_dim] on the device, see `scales_ptr`): the fp8 side's
    dequantisation scale per (layer, outer), applied by the cast.  include/kvbm_kernels.h (kvbm_kernels_paged_permute_heads,
    kvbm_kernels_paged_permute_heads_scaled)."""
    if cast_scales is not None:
        return lib().kvbm_kernels_paged_permute_heads_scaled(C.byref(src), C.byref(dst), num_blocks, layer_begin, layer_end, src_num_heads,
                                                             src_head_begin, dst_num_heads, dst_head_begin, head_count, page_size,
                                                             src_row_bytes, int(cast_mode), scales_ptr(cast_scales), done_flag or None, epoch,
                                                             completion_flag or None, completion_value, stream)
    return lib().kvbm_kernels_paged_permute_heads(C.byref(src), C.byref(dst), num_blocks, layer_begin, layer_end, src_num_heads,
                                                  src_head_begin, dst_num_heads, dst_head_begin, head_count, page_size, src_row_bytes,
                                                  int(cast_mode), done_flag or None, epoch, completion_flag or None, completion_value, stream)


def paged_permute_gather(srcs: Sequence[PermuteSource], dst: PermuteSide, dst_num_heads: int, num_blocks: int, layer_begin: int,
                         layer_end: int, page_size: int, src_row_bytes: int, cast_mode: int = 0, done_flag: int = 0, epoch: int = 0,
                         completion_flag: int = 0, completion_value: int = 0, stream: int = 0, cast_scales=None) -> int:
    """`paged_permute_heads` over several sources in ONE launch (a TP re-shard's assembly): each source's head window lands in
    the destination, whose bytes outside the union of the windows keep their values; the flags are written once, after every
    window.  `cast_scales`: one scale array for every source, as `paged_permute_heads`.  include/kvbm_kernels.h
    (kvbm_kernels_paged_permute_gather, kvbm_kernels_paged_permute_gather_scaled)."""
    arr = (PermuteSource * max(1, len(srcs)))(*srcs)
    if cast_scales is not None:
        return lib().kvbm_kernels_paged_permute_gather_scaled(arr, len(srcs), C.byref(dst), dst_num_heads, num_blocks, layer_begin, layer_end,
                                                              page_size, src_row_bytes, int(cast_mode), scales_ptr(cast_scales),
                                                              done_flag or None, epoch, completion_flag or None, completion_value, stream)
    return lib().kvbm_kernels_paged_permute_gather(arr, len(srcs), C.byref(dst), dst_num_heads, num_blocks, layer_begin, layer_end, page_size,
                                                   src_row_bytes, int(cast_mode), done_flag or None, epoch, completion_flag or None,
                                                   completion_value, stream)


def paged_repage(src: PermuteSide, src_page_size: int, dst: PermuteSide, dst_page_size: int, token_begin: int, token_end: int,
                 layer_begin: int, layer_end: int, num_heads: int, src_row_bytes: int, cast_mode: int = 0, cast_scales=None,
                 done_flag: int = 0, epoch: int = 0, completion_flag: int = 0, completion_value: int = 0, stream: int = 0) -> int:
    """Tokens [token_begin, token_end) of one sequence between two block tables with different page sizes (one divides the other):
    src.block_ids = src_table[token_begin // Ps .. ceil(token_end / Ps)), dst.block_ids likewise for Pd; re-ordered between the
    formats and cast as `paged_permute_heads` would; every other destination byte keeps its value.  include/kvbm_kernels.h
    (kvbm_kernels_paged_repage)."""
    return lib().kvbm_kernels_paged_repage(C.byref(src), src_page_size, C.byref(dst), dst_page_size, token_begin, token_end, layer_begin,
                                           layer_end, num_heads, src_row_bytes, int(cast_mode), scales_ptr(cast_scales), done_flag or None,
                                           epoch, completion_flag or None, completion_value, stream)


def paged_repage_gather(srcs: Sequence[PermuteSource], src_page_size: int, dst: PermuteSide, dst_num_heads: int, dst_page_size: int,
                        token_begin: int, token_end: int, layer_begin: int, layer_end: int, src_row_bytes: int, cast_mode: int = 0,
                        cast_scales=None, done_flag: int = 0, epoch: int = 0, completion_flag: int = 0, completion_value: int = 0,
                        stream: int = 0) -> int:
    """`paged_permute_gather`'s head windows over `paged_repage`'s token range, in ONE launch: every source shares the page size
    src_page_size (its block_ids = its table[token_begin // Ps .. ceil(token_end / Ps))), the destination has its own
    (dst.block_ids likewise for Pd); every destination byte outside the windows' heads and the range keeps its value, and the
    flags are written once.  include/kvbm_kernels.h (kvbm_kernels_paged_repage_gather)."""
    arr = (PermuteSource * max(1, len(srcs)))(*srcs)
    return lib().kvbm_kernels_paged_repage_gather(arr, len(srcs), src_page_size, C.byref(dst), dst_num_heads, dst_page_size, token_begin,
                                                  token_end, layer_begin, layer_end, src_row_bytes, int(cast_mode), scales_ptr(cast_scales),
                                                  done_flag or None, epoch, completion_flag or None, completion_value, stream)


def paged_permute_gather_streamed(srcs: Sequence[PermuteSource], dst: PermuteSide, dst_num_heads: int, num_blocks: int, layer_begin: int,
                                  layer_end: int, page_size: int, src_row_bytes: int, cast_mode: int, cast_scales,
                                  st: Optional[PermuteStream], stream: int = 0) -> int:
    """`paged_permute_gather` streamed layer by layer behind `st`'s ready flags (one array per source); the flags of `st` replace the
    done / completion arguments.  One source with a full window is a format change, one with a partial window a re-shard.
    include/kvbm_kernels.h (kvbm_kernels_paged_permute_gather_streamed)."""
    arr = (PermuteSource * max(1, len(srcs)))(*srcs)
    return lib().kvbm_kernels_paged_permute_gather_streamed(arr, len(srcs), C.byref(dst), dst_num_heads, num_blocks, layer_begin, layer_end,
                                                            page_size, src_row_bytes, int(cast_mode), scales_ptr(cast_scales),
                                                            C.byref(st) if st is not None else None, stream)


def paged_repage_gather_streamed(srcs: Sequence[PermuteSource], src_page_size: int, dst: PermuteSide, dst_num_heads: int,
                                 dst_page_size: int, token_begin: int, token_end: int, layer_begin: int, layer_end: int, src_row_bytes: int,
                                 cast_mode: int, cast_scales, st: Optional[PermuteStream], stream: int = 0) -> int:
    """`paged_repage_gather` streamed as `paged_permute_gather_streamed`; one full-window source is `paged_repage`.
    include/kvbm_kernels.h (kvbm_kernels_paged_repage_gather_streamed)."""
    arr = (PermuteSource * max(1, len(srcs)))(*srcs)
    return lib().kvbm_kernels_paged_repage_gather_streamed(arr, len(srcs), src_page_size, C.byref(dst), dst_num_heads, dst_page_size,
                                                           token_begin, token_end, layer_begin, layer_end, src_row_bytes, int(cast_mode),
                                                           scales_ptr(cast_scales), C.byref(st) if st is not None else None, stream)


def paged_stage_gather(srcs: Sequence[StageSource], dst: PermuteSide, dst_num_heads: int, num_blocks: int, layer_begin: int,
                       layer_end: int, page_size: int, src_row_bytes: int, cast_mode: int = 0, cast_scales=None, done_flag: int = 0,
                       epoch: int = 0, completion_flag: int = 0, completion_value: int = 0, stream: int = 0) -> int:
    """`paged_permute_gather` with a layer window per source, in ONE launch (a decode rank assembling its layers and heads from a
    PP x TP prefill group): sources with equal destination layer windows form a stage, and every destination layer of
    [layer_begin, layer_end) takes the head windows of its stage, each read at the source's own layer.  `cast_scales` is indexed
    by the destination layer.  include/kvbm_kernels.h (kvbm_kernels_paged_stage_gather)."""
    arr = (StageSource * max(1, len(srcs)))(*srcs)
    return lib().kvbm_kernels_paged_stage_gather(arr, len(srcs), C.byref(dst), dst_num_heads, num_blocks, layer_begin, layer_end, page_size,
                                                 src_row_bytes, int(cast_mode), scales_ptr(cast_scales), done_flag or None, epoch,
                                                 completion_flag or None, completion_value, stream)


def paged_stage_gather_streamed(srcs: Sequence[StageSource], dst: PermuteSide, dst_num_heads: int, num_blocks: int, layer_begin: int,
                                layer_end: int, page_size: int, src_row_bytes: int, cast_mode: int, cast_scales,
                                st: Optional[PermuteStream], stream: int = 0) -> int:
    """`paged_stage_gather` streamed layer by layer: `st.layer_ready_flags[s]` is source s's array over its own layers, and a
    destination layer waits only for the sources of its stage.  include/kvbm_kernels.h (kvbm_kernels_paged_stage_gather_streamed)."""
    arr = (StageSource * max(1, len(srcs)))(*srcs)
    return lib().kvbm_kernels_paged_stage_gather_streamed(arr, len(srcs), C.byref(dst), dst_num_heads, num_blocks, layer_begin, layer_end,
                                                          page_size, src_row_bytes, int(cast_mode), scales_ptr(cast_scales),
                                                          C.byref(st) if st is not None else None, stream)


def paged_stage_repage_gather(srcs: Sequence[StageSource], src_page_size: int, dst: PermuteSide, dst_num_heads: int, dst_page_size: int,
                              token_begin: int, token_end: int, layer_begin: int, layer_end: int, src_row_bytes: int, cast_mode: int = 0,
                              cast_scales=None, done_flag: int = 0, epoch: int = 0, completion_flag: int = 0, completion_value: int = 0,
                              stream: int = 0) -> int:
    """`paged_stage_gather`'s layer windows over `paged_repage_gather`'s token range, in ONE launch (a decode rank assembling its
    layers and heads from a PP x TP prefill group with another page size): every source shares src_page_size and its block_ids
    are its table[token_begin // Ps .. ceil(token_end / Ps)); `cast_scales` is indexed by the destination layer.
    include/kvbm_kernels.h (kvbm_kernels_paged_stage_repage_gather)."""
    arr = (StageSource * max(1, len(srcs)))(*srcs)
    return lib().kvbm_kernels_paged_stage_repage_gather(arr, len(srcs), src_page_size, C.byref(dst), dst_num_heads, dst_page_size,
                                                        token_begin, token_end, layer_begin, layer_end, src_row_bytes, int(cast_mode),
                                                        scales_ptr(cast_scales), done_flag or None, epoch, completion_flag or None,
                                                        completion_value, stream)


def paged_stage_repage_gather_streamed(srcs: Sequence[StageSource], src_page_size: int, dst: PermuteSide, dst_num_heads: int,
                                       dst_page_size: int, token_begin: int, token_end: int, layer_begin: int, layer_end: int,
                                       src_row_bytes: int, cast_mode: int, cast_scales, st: Optional[PermuteStream],
                                       stream: int = 0) -> int:
    """`paged_stage_repage_gather` streamed with `paged_stage_gather_streamed`'s flags: `st.layer_ready_flags[s]` runs over source
    s's own layers.  include/kvbm_kernels.h (kvbm_kernels_paged_stage_repage_gather_streamed)."""
    arr = (StageSource * max(1, len(srcs)))(*srcs)
    return lib().kvbm_kernels_paged_stage_repage_gather_streamed(arr, len(srcs), src_page_size, C.byref(dst), dst_num_heads, dst_page_size,
                                                                 token_begin, token_end, layer_begin, layer_end, src_row_bytes,
                                                                 int(cast_mode), scales_ptr(cast_scales),
                                                                 C.byref(st) if st is not None else None, stream)


def _repage_seqs(seqs: Sequence[Tuple[int, int]]):
    return (RepageSeq * max(1, len(seqs)))(*[RepageSeq(int(b), int(e)) for b, e in seqs])


def _unit_table(call, arr, num_seqs: int, src_page_size: int, dst_page_size: int):
    """A unit helper's sizing call, then its table as a numpy uint32 array [num_units, 4] with the two table lengths, or None."""
    import numpy as np
    n, ns, nd = C.c_size_t(), C.c_size_t(), C.c_size_t()
    if call(C.cast(arr, C.c_void_p), num_seqs, src_page_size, dst_page_size, None, 0, C.byref(n), C.byref(ns), C.byref(nd)):
        return None
    out = np.zeros((n.value, 4), dtype=np.uint32)
    if call(C.cast(arr, C.c_void_p), num_seqs, src_page_size, dst_page_size, out.ctypes.data, n.value, C.byref(n), C.byref(ns), C.byref(nd)):
        return None
    return out, ns.value, nd.value


def repage_batch_units(seqs: Sequence[Tuple[int, int]], src_page_size: int, dst_page_size: int):
    """Host-only: the unit table of a batch of (token_begin, token_end) ranges as a numpy uint32 array [num_units, 4] (q0, tokens,
    small_k, seq) and the lengths of each source's and the destination's concatenated block table; None when the pages or a range
    break a rule.  include/kvbm_kernels.h (kvbm_kernels_repage_batch_units)."""
    return _unit_table(lib().kvbm_kernels_repage_batch_units, _repage_seqs(seqs), len(seqs), src_page_size, dst_page_size)


def paged_stage_repage_gather_batch(srcs: Sequence[StageSource], src_page_size: int, dst: PermuteSide, dst_num_heads: int,
                                    dst_page_size: int, seqs: Sequence[Tuple[int, int]], units: int, num_units: int, layer_begin: int,
                                    layer_end: int, src_row_bytes: int, cast_mode: int = 0, cast_scales=None, done_flag: int = 0,
                                    epoch: int = 0, completion_flag: int = 0, completion_value: int = 0, stream: int = 0) -> int:
    """`paged_stage_repage_gather` over a batch of sequences in ONE launch with one signal: `seqs` are the (token_begin, token_end)
    ranges, every side's block_ids the concatenation of the per-sequence tables, `units` the device address of the table
    `repage_batch_units` made for the same ranges and pages.  Two sequences must not share a destination block.
    include/kvbm_kernels.h (kvbm_kernels_paged_stage_repage_gather_batch)."""
    arr = (StageSource * max(1, len(srcs)))(*srcs)
    return lib().kvbm_kernels_paged_stage_repage_gather_batch(arr, len(srcs), src_page_size, C.byref(dst), dst_num_heads, dst_page_size,
                                                              C.cast(_repage_seqs(seqs), C.c_void_p), len(seqs), units or None, num_units,
                                                              layer_begin, layer_end, src_row_bytes, int(cast_mode),
                                                              scales_ptr(cast_scales), done_flag or None, epoch, completion_flag or None,
                                                              completion_value, stream)


def paged_stage_repage_gather_batch_streamed(srcs: Sequence[StageSource], src_page_size: int, dst: PermuteSide, dst_num_heads: int,
                                             dst_page_size: int, seqs: Sequence[Tuple[int, int]], units: int, num_units: int,
                                             layer_begin: int, layer_end: int, src_row_bytes: int, cast_mode: int, cast_scales,
                                             st: Optional[PermuteStream], stream: int = 0) -> int:
    """`paged_stage_repage_gather_batch` streamed with `paged_stage_repage_gather_streamed`'s flags: one ready flag per (source,
    layer) covers the batch.  include/kvbm_kernels.h (kvbm_kernels_paged_stage_repage_gather_batch_streamed)."""
    arr = (StageSource * max(1, len(srcs)))(*srcs)
    return lib().kvbm_kernels_paged_stage_repage_gather_batch_streamed(arr, len(srcs), src_page_size, C.byref(dst), dst_num_heads,
                                                                       dst_page_size, C.cast(_repage_seqs(seqs), C.c_void_p), len(seqs),
                                                                       units or None, num_units, layer_begin, layer_end, src_row_bytes,
                                                                       int(cast_mode), scales_ptr(cast_scales),
                                                                       C.byref(st) if st is not None else None, stream)


def repage_anypage_units(seqs: Sequence[Tuple[int, int]], src_page_size: int, dst_page_size: int):
    """Host-only: `repage_batch_units` for any two non-zero pages, each record's fourth word its big block's phase (the slot of
    small block small_k that holds the big block's slot 0): a numpy uint32 array [num_units, 4] (q0, tokens, small_k, phase) and
    the two table lengths, or None when the pages pass the exactness bound or a range breaks a rule.
    include/kvbm_kernels.h (kvbm_kernels_repage_anypage_units)."""
    return _unit_table(lib().kvbm_kernels_repage_anypage_units, _repage_seqs(seqs), len(seqs), src_page_size, dst_page_size)


def paged_stage_repage_gather_anypage(srcs: Sequence[StageSource], src_page_size: int, dst: PermuteSide, dst_num_heads: int,
                                      dst_page_size: int, seqs: Sequence[Tuple[int, int]], units: int, num_units: int, layer_begin: int,
                                      layer_end: int, src_row_bytes: int, cast_mode: int = 0, cast_scales=None, done_flag: int = 0,
                                      epoch: int = 0, completion_flag: int = 0, completion_value: int = 0, stream: int = 0) -> int:
    """`paged_stage_repage_gather_batch` for any two non-zero pages, dividing or not: `units` is the device address of the table
    `repage_anypage_units` made for the same ranges and pages.  With dividing pages it writes the batch's bytes.
    include/kvbm_kernels.h (kvbm_kernels_paged_stage_repage_gather_anypage)."""
    arr = (StageSource * max(1, len(srcs)))(*srcs)
    return lib().kvbm_kernels_paged_stage_repage_gather_anypage(arr, len(srcs), src_page_size, C.byref(dst), dst_num_heads, dst_page_size,
                                                                C.cast(_repage_seqs(seqs), C.c_void_p), len(seqs), units or None, num_units,
                                                                layer_begin, layer_end, src_row_bytes, int(cast_mode),
                                                                scales_ptr(cast_scales), done_flag or None, epoch, completion_flag or None,
                                                                completion_value, stream)


def paged_stage_repage_gather_anypage_streamed(srcs: Sequence[StageSource], src_page_size: int, dst: PermuteSide, dst_num_heads: int,
                                               dst_page_size: int, seqs: Sequence[Tuple[int, int]], units: int, num_units: int,
                                               layer_begin: int, layer_end: int, src_row_bytes: int, cast_mode: int, cast_scales,
                                               st: Optional[PermuteStream], stream: int = 0) -> int:
    """`paged_stage_repage_gather_anypage` streamed with `paged_stage_repage_gather_batch_streamed`'s flags and gate forms.
    include/kvbm_kernels.h (kvbm_kernels_paged_stage_repage_gather_anypage_streamed)."""
    arr = (StageSource * max(1, len(srcs)))(*srcs)
    return lib().kvbm_kernels_paged_stage_repage_gather_anypage_streamed(arr, len(srcs), src_page_size, C.byref(dst), dst_num_heads,
                                                                         dst_page_size, C.cast(_repage_seqs(seqs), C.c_void_p), len(seqs),
                                                                         units or None, num_units, layer_begin, layer_end, src_row_bytes,
                                                                         int(cast_mode), scales_ptr(cast_scales),
                                                                         C.byref(st) if st is not None else None, stream)


def paged_repage_scatter(src: PermuteSide, src_num_heads: int, src_page_size: int, targets: Sequence[ScatterTarget], dst_page_size: int,
                         token_begin: int, token_end: int, layer_begin: int, layer_end: int, src_row_bytes: int, cast_mode: int = 0,
                         cast_scales=None, epoch: int = 0, completion_flag: int = 0, completion_value: int = 0, stream: int = 0) -> int:
    """One source (its block_ids = its table[token_begin // Ps .. ceil(token_end / Ps))) into every target in ONE launch: each
    target's head window of the source's layer window lands in its destination at its own heads and layers, every source vector
    read once and cast once; the layer range and `cast_scales` count SOURCE layers.  Then every target's done flag (epoch) and the
    completion word are written once.  include/kvbm_kernels.h (kvbm_kernels_paged_repage_scatter)."""
    arr = (ScatterTarget * max(1, len(targets)))(*targets)
    return lib().kvbm_kernels_paged_repage_scatter(C.byref(src), src_num_heads, src_page_size, arr, len(targets), dst_page_size, token_begin,
                                                   token_end, layer_begin, layer_end, src_row_bytes, int(cast_mode), scales_ptr(cast_scales),
                                                   epoch, completion_flag or None, completion_value, stream)


def paged_repage_scatter_streamed(src: PermuteSide, src_num_heads: int, src_page_size: int, targets: Sequence[ScatterTarget],
                                  dst_page_size: int, token_begin: int, token_end: int, layer_begin: int, layer_end: int,
                                  src_row_bytes: int, cast_mode: int, cast_scales, st: Optional[PermuteStream], stream: int = 0) -> int:
    """`paged_repage_scatter` streamed layer by layer behind the source's ready flags: `st.layer_ready_flags[0]` is the source's
    [num_layers] array, and source layer l is read only once its flag reaches `st.epoch`.  `st.layer_done_flags` and
    `st.sync_workspace` count source layers; `st.epoch` is also what every target's done flag receives.  The bytes are the
    unstreamed call's.  include/kvbm_kernels.h (kvbm_kernels_paged_repage_scatter_streamed)."""
    arr = (ScatterTarget * max(1, len(targets)))(*targets)
    return lib().kvbm_kernels_paged_repage_scatter_streamed(C.byref(src), src_num_heads, src_page_size, arr, len(targets), dst_page_size,
                                                            token_begin, token_end, layer_begin, layer_end, src_row_bytes, int(cast_mode),
                                                            scales_ptr(cast_scales), C.byref(st) if st is not None else None, stream)


def paged_repage_scatter_batch(src: PermuteSide, src_num_heads: int, src_page_size: int, targets: Sequence[ScatterTarget],
                               dst_page_size: int, seqs: Sequence[Tuple[int, int]], units: int, num_units: int, layer_begin: int,
                               layer_end: int, src_row_bytes: int, cast_mode: int = 0, cast_scales=None, epoch: int = 0,
                               completion_flag: int = 0, completion_value: int = 0, stream: int = 0) -> int:
    """`paged_repage_scatter` over a batch of sequences in ONE launch with one signal: `seqs` are the (token_begin, token_end)
    ranges, the source's and every target's block_ids the concatenation of the per-sequence tables, `units` the device address of
    the table `repage_batch_units` made for the same ranges and pages (Ps, Pd).  Two sequences must not share a destination block
    of one target pool.  include/kvbm_kernels.h (kvbm_kernels_paged_repage_scatter_batch)."""
    arr = (ScatterTarget * max(1, len(targets)))(*targets)
    return lib().kvbm_kernels_paged_repage_scatter_batch(C.byref(src), src_num_heads, src_page_size, arr, len(targets), dst_page_size,
                                                         C.cast(_repage_seqs(seqs), C.c_void_p), len(seqs), units or None, num_units,
                                                         layer_begin, layer_end, src_row_bytes, int(cast_mode), scales_ptr(cast_scales),
                                                         epoch, completion_flag or None, completion_value, stream)


def paged_repage_scatter_batch_streamed(src: PermuteSide, src_num_heads: int, src_page_size: int, targets: Sequence[ScatterTarget],
                                        dst_page_size: int, seqs: Sequence[Tuple[int, int]], units: int, num_units: int,
                                        layer_begin: int, layer_end: int, src_row_bytes: int, cast_mode: int, cast_scales,
                                        st: Optional[PermuteStream], stream: int = 0) -> int:
    """`paged_repage_scatter_batch` streamed with `paged_repage_scatter_streamed`'s flags: one ready flag per source layer covers
    the batch, and layer_done_flags[l] is written once source layer l of every sequence landed in every target.
    include/kvbm_kernels.h (kvbm_kernels_paged_repage_scatter_batch_streamed)."""
    arr = (ScatterTarget * max(1, len(targets)))(*targets)
    return lib().kvbm_kernels_paged_repage_scatter_batch_streamed(C.byref(src), src_num_heads, src_page_size, arr, len(targets),
                                                                  dst_page_size, C.cast(_repage_seqs(seqs), C.c_void_p), len(seqs),
                                                                  units or None, num_units, layer_begin, layer_end, src_row_bytes,
                                                                  int(cast_mode), scales_ptr(cast_scales),
                                                                  C.byref(st) if st is not None else None, stream)


def paged_repage_scatter_anypage(src: PermuteSide, src_num_heads: int, src_page_size: int, targets: Sequence[ScatterTarget],
                                 dst_page_size: int, seqs: Sequence[Tuple[int, int]], units: int, num_units: int, layer_begin: int,
                                 layer_end: int, src_row_bytes: int, cast_mode: int = 0, cast_scales=None, epoch: int = 0,
                                 completion_flag: int = 0, completion_value: int = 0, stream: int = 0) -> int:
    """`paged_repage_scatter_batch` for any two non-zero pages, dividing or not: `units` is the device address of the table
    `repage_anypage_units` made for the same ranges and pages (Ps, Pd), which serves every target.  With dividing pages it writes
    the batch scatter's bytes.  include/kvbm_kernels.h (kvbm_kernels_paged_repage_scatter_anypage)."""
    arr = (ScatterTarget * max(1, len(targets)))(*targets)
    return lib().kvbm_kernels_paged_repage_scatter_anypage(C.byref(src), src_num_heads, src_page_size, arr, len(targets), dst_page_size,
                                                           C.cast(_repage_seqs(seqs), C.c_void_p), len(seqs), units or None, num_units,
                                                           layer_begin, layer_end, src_row_bytes, int(cast_mode), scales_ptr(cast_scales),
                                                           epoch, completion_flag or None, completion_value, stream)


def paged_repage_scatter_anypage_streamed(src: PermuteSide, src_num_heads: int, src_page_size: int, targets: Sequence[ScatterTarget],
                                          dst_page_size: int, seqs: Sequence[Tuple[int, int]], units: int, num_units: int,
                                          layer_begin: int, layer_end: int, src_row_bytes: int, cast_mode: int, cast_scales,
                                          st: Optional[PermuteStream], stream: int = 0) -> int:
    """`paged_repage_scatter_anypage` streamed with `paged_repage_scatter_batch_streamed`'s flags and gate forms.
    include/kvbm_kernels.h (kvbm_kernels_paged_repage_scatter_anypage_streamed)."""
    arr = (ScatterTarget * max(1, len(targets)))(*targets)
    return lib().kvbm_kernels_paged_repage_scatter_anypage_streamed(C.byref(src), src_num_heads, src_page_size, arr, len(targets),
                                                                    dst_page_size, C.cast(_repage_seqs(seqs), C.c_void_p), len(seqs),
                                                                    units or None, num_units, layer_begin, layer_end, src_row_bytes,
                                                                    int(cast_mode), scales_ptr(cast_scales),
                                                                    C.byref(st) if st is not None else None, stream)


def _route_seqs(seqs: Sequence[Tuple[int, int, int]]):
    return (RouteSeq * max(1, len(seqs)))(*[RouteSeq(int(b), int(e), int(t)) for b, e, t in seqs])


def repage_route_units(seqs: Sequence[Tuple[int, int, int]], src_page_size: int, dst_page_size: int):
    """Host-only: `repage_batch_units` over the (token_begin, token_end, targets) of a routed batch, each record's fourth word its
    sequence's targets: a numpy uint32 array [num_units, 4] (q0, tokens, small_k, targets) and the two table lengths, or None.
    include/kvbm_kernels.h (kvbm_kernels_repage_route_units)."""
    return _unit_table(lib().kvbm_kernels_repage_route_units, _route_seqs(seqs), len(seqs), src_page_size, dst_page_size)


def paged_repage_scatter_routed(src: PermuteSide, src_num_heads: int, src_page_size: int, targets: Sequence[ScatterTarget],
                                dst_page_size: int, seqs: Sequence[Tuple[int, int, int]], units: int, num_units: int, layer_begin: int,
                                layer_end: int, src_row_bytes: int, cast_mode: int = 0, cast_scales=None, epoch: int = 0,
                                completion_flag: int = 0, completion_value: int = 0, stream: int = 0) -> int:
    """`paged_repage_scatter_batch` with a target mask per sequence, in ONE launch with one signal: `seqs` are (token_begin,
    token_end, targets), bit t of targets naming targets[t]; every target's block_ids has the batch layout (the positions of
    sequences not routed to it are never read); `units` is the device address of the table `repage_route_units` made for the same
    sequences and pages.  include/kvbm_kernels.h (kvbm_kernels_paged_repage_scatter_routed)."""
    arr = (ScatterTarget * max(1, len(targets)))(*targets)
    return lib().kvbm_kernels_paged_repage_scatter_routed(C.byref(src), src_num_heads, src_page_size, arr, len(targets), dst_page_size,
                                                          C.cast(_route_seqs(seqs), C.c_void_p), len(seqs), units or None, num_units,
                                                          layer_begin, layer_end, src_row_bytes, int(cast_mode), scales_ptr(cast_scales),
                                                          epoch, completion_flag or None, completion_value, stream)


def paged_repage_scatter_routed_streamed(src: PermuteSide, src_num_heads: int, src_page_size: int, targets: Sequence[ScatterTarget],
                                         dst_page_size: int, seqs: Sequence[Tuple[int, int, int]], units: int, num_units: int,
                                         layer_begin: int, layer_end: int, src_row_bytes: int, cast_mode: int, cast_scales,
                                         st: Optional[PermuteStream], stream: int = 0) -> int:
    """`paged_repage_scatter_routed` streamed with `paged_repage_scatter_batch_streamed`'s flags: layer_done_flags[l] is written
    once source layer l of every sequence landed in every target it is routed to.
    include/kvbm_kernels.h (kvbm_kernels_paged_repage_scatter_routed_streamed)."""
    arr = (ScatterTarget * max(1, len(targets)))(*targets)
    return lib().kvbm_kernels_paged_repage_scatter_routed_streamed(C.byref(src), src_num_heads, src_page_size, arr, len(targets),
                                                                   dst_page_size, C.cast(_route_seqs(seqs), C.c_void_p), len(seqs),
                                                                   units or None, num_units, layer_begin, layer_end, src_row_bytes,
                                                                   int(cast_mode), scales_ptr(cast_scales),
                                                                   C.byref(st) if st is not None else None, stream)


def paged_stage_repage_gather_routed(srcs: Sequence[StageSource], src_page_size: int, dst: PermuteSide, dst_num_heads: int,
                                     dst_page_size: int, seqs: Sequence[Tuple[int, int, int]], units: int, num_units: int, layer_begin: int,
                                     layer_end: int, src_row_bytes: int, cast_mode: int = 0, cast_scales=None, done_flag: int = 0,
                                     epoch: int = 0, completion_flag: int = 0, completion_value: int = 0, stream: int = 0) -> int:
    """`paged_stage_repage_gather_batch` with a source mask per sequence, in ONE launch with one signal: `seqs` are (token_begin,
    token_end, sources), bit s of sources naming srcs[s]; every source's block_ids has the batch layout (the positions of sequences
    not routed to it are never read); `units` is the device address of the table `repage_route_units` made for the same sequences
    and pages.  Two windows of a stage may share destination heads when no mask holds both.
    include/kvbm_kernels.h (kvbm_kernels_paged_stage_repage_gather_routed)."""
    arr = (StageSource * max(1, len(srcs)))(*srcs)
    return lib().kvbm_kernels_paged_stage_repage_gather_routed(arr, len(srcs), src_page_size, C.byref(dst), dst_num_heads, dst_page_size,
                                                               C.cast(_route_seqs(seqs), C.c_void_p), len(seqs), units or None, num_units,
                                                               layer_begin, layer_end, src_row_bytes, int(cast_mode),
                                                               scales_ptr(cast_scales), done_flag or None, epoch, completion_flag or None,
                                                               completion_value, stream)


def paged_stage_repage_gather_routed_streamed(srcs: Sequence[StageSource], src_page_size: int, dst: PermuteSide, dst_num_heads: int,
                                              dst_page_size: int, seqs: Sequence[Tuple[int, int, int]], units: int, num_units: int,
                                              layer_begin: int, layer_end: int, src_row_bytes: int, cast_mode: int, cast_scales,
                                              st: Optional[PermuteStream], stream: int = 0) -> int:
    """`paged_stage_repage_gather_routed` streamed with `paged_stage_repage_gather_batch_streamed`'s flags; only the sources some
    sequence is routed to are waited on, and the others' ready flags may be 0.
    include/kvbm_kernels.h (kvbm_kernels_paged_stage_repage_gather_routed_streamed)."""
    arr = (StageSource * max(1, len(srcs)))(*srcs)
    return lib().kvbm_kernels_paged_stage_repage_gather_routed_streamed(arr, len(srcs), src_page_size, C.byref(dst), dst_num_heads,
                                                                        dst_page_size, C.cast(_route_seqs(seqs), C.c_void_p), len(seqs),
                                                                        units or None, num_units, layer_begin, layer_end, src_row_bytes,
                                                                        int(cast_mode), scales_ptr(cast_scales),
                                                                        C.byref(st) if st is not None else None, stream)


def repage_route_anypage_units(seqs: Sequence[Tuple[int, int, int]], src_page_size: int, dst_page_size: int):
    """Host-only: `repage_anypage_units` over the (token_begin, token_end, targets) of a routed batch, each record's fourth word its
    sequence's targets | its block's phase << 16: a numpy uint32 array [num_units, 4] (q0, tokens, small_k, route) and the two table
    lengths, or None (also for a mask with a bit at or above 16).  include/kvbm_kernels.h (kvbm_kernels_repage_route_anypage_units)."""
    return _unit_table(lib().kvbm_kernels_repage_route_anypage_units, _route_seqs(seqs), len(seqs), src_page_size, dst_page_size)


def paged_repage_scatter_routed_anypage(src: PermuteSide, src_num_heads: int, src_page_size: int, targets: Sequence[ScatterTarget],
                                        dst_page_size: int, seqs: Sequence[Tuple[int, int, int]], units: int, num_units: int,
                                        layer_begin: int, layer_end: int, src_row_bytes: int, cast_mode: int = 0, cast_scales=None,
                                        epoch: int = 0, completion_flag: int = 0, completion_value: int = 0, stream: int = 0) -> int:
    """`paged_repage_scatter_routed` for any two non-zero pages, dividing or not: `units` is the device address of the table
    `repage_route_anypage_units` made for the same sequences and pages.  include/kvbm_kernels.h
    (kvbm_kernels_paged_repage_scatter_routed_anypage)."""
    arr = (ScatterTarget * max(1, len(targets)))(*targets)
    return lib().kvbm_kernels_paged_repage_scatter_routed_anypage(C.byref(src), src_num_heads, src_page_size, arr, len(targets),
                                                                  dst_page_size, C.cast(_route_seqs(seqs), C.c_void_p), len(seqs),
                                                                  units or None, num_units, layer_begin, layer_end, src_row_bytes,
                                                                  int(cast_mode), scales_ptr(cast_scales), epoch, completion_flag or None,
                                                                  completion_value, stream)


def paged_repage_scatter_routed_anypage_streamed(src: PermuteSide, src_num_heads: int, src_page_size: int,
                                                 targets: Sequence[ScatterTarget], dst_page_size: int, seqs: Sequence[Tuple[int, int, int]],
                                                 units: int, num_units: int, layer_begin: int, layer_end: int, src_row_bytes: int,
                                                 cast_mode: int, cast_scales, st: Optional[PermuteStream], stream: int = 0) -> int:
    """`paged_repage_scatter_routed_anypage` streamed with `paged_repage_scatter_routed_streamed`'s flags and gate forms.
    include/kvbm_kernels.h (kvbm_kernels_paged_repage_scatter_routed_anypage_streamed)."""
    arr = (ScatterTarget * max(1, len(targets)))(*targets)
    return lib().kvbm_kernels_paged_repage_scatter_routed_anypage_streamed(C.byref(src), src_num_heads, src_page_size, arr, len(targets),
                                                                           dst_page_size, C.cast(_route_seqs(seqs), C.c_void_p), len(seqs),
                                                                           units or None, num_units, layer_begin, layer_end, src_row_bytes,
                                                                           int(cast_mode), scales_ptr(cast_scales),
                                                                           C.byref(st) if st is not None else None, stream)


def paged_stage_repage_gather_routed_anypage(srcs: Sequence[StageSource], src_page_size: int, dst: PermuteSide, dst_num_heads: int,
                                             dst_page_size: int, seqs: Sequence[Tuple[int, int, int]], units: int, num_units: int,
                                             layer_begin: int, layer_end: int, src_row_bytes: int, cast_mode: int = 0, cast_scales=None,
                                             done_flag: int = 0, epoch: int = 0, completion_flag: int = 0, completion_value: int = 0,
                                             stream: int = 0) -> int:
    """`paged_stage_repage_gather_routed` for any two non-zero pages, dividing or not: `units` is the device address of the table
    `repage_route_anypage_units` made for the same sequences and pages.  include/kvbm_kernels.h
    (kvbm_kernels_paged_stage_repage_gather_routed_anypage)."""
    arr = (StageSource * max(1, len(srcs)))(*srcs)
    return lib().kvbm_kernels_paged_stage_repage_gather_routed_anypage(arr, len(srcs), src_page_size, C.byref(dst), dst_num_heads,
                                                                       dst_page_size, C.cast(_route_seqs(seqs), C.c_void_p), len(seqs),
                                                                       units or None, num_units, layer_begin, layer_end, src_row_bytes,
                                                                       int(cast_mode), scales_ptr(cast_scales), done_flag or None, epoch,
                                                                       completion_flag or None, completion_value, stream)


def paged_stage_repage_gather_routed_anypage_streamed(srcs: Sequence[StageSource], src_page_size: int, dst: PermuteSide,
                                                      dst_num_heads: int, dst_page_size: int, seqs: Sequence[Tuple[int, int, int]],
                                                      units: int, num_units: int, layer_begin: int, layer_end: int, src_row_bytes: int,
                                                      cast_mode: int, cast_scales, st: Optional[PermuteStream], stream: int = 0) -> int:
    """`paged_stage_repage_gather_routed_anypage` streamed with `paged_stage_repage_gather_routed_streamed`'s flags and gate forms;
    only the sources some sequence is routed to are waited on.
    include/kvbm_kernels.h (kvbm_kernels_paged_stage_repage_gather_routed_anypage_streamed)."""
    arr = (StageSource * max(1, len(srcs)))(*srcs)
    return lib().kvbm_kernels_paged_stage_repage_gather_routed_anypage_streamed(arr, len(srcs), src_page_size, C.byref(dst), dst_num_heads,
                                                                                dst_page_size, C.cast(_route_seqs(seqs), C.c_void_p),
                                                                                len(seqs), units or None, num_units, layer_begin, layer_end,
                                                                                src_row_bytes, int(cast_mode), scales_ptr(cast_scales),
                                                                                C.byref(st) if st is not None else None, stream)


def permute_strides(kv_layout: int, num_layers: int, outer_dim: int, num_heads: int, page_size: int, row_bytes: int,
                    block_stride: int, outer_stride: int):
    """Host-only: (universal, layer_step, outer_step, head_stride, tok_stride) of one side of `paged_permute`, or None."""
    out = (C.c_uint64 * 5)()
    if lib().kvbm_kernels_permute_strides(int(kv_layout), num_layers, outer_dim, num_heads, page_size, row_bytes, block_stride,
                                          outer_stride, out):
        return None
    return bool(out[0]), int(out[1]), int(out[2]), int(out[3]), int(out[4])


def set_flags(flags_ptr: int, first: int, count: int, value: int, stream: int) -> int:
    return lib().kvbm_kernels_set_flags(flags_ptr, first, count, value, stream)


def stream_wait_event(stream: int, event: int) -> int:
    return lib().kvbm_kernels_stream_wait_event(stream, event)


def wait_flag(flag_ptr: int, value: int, stream: int) -> int:
    return lib().kvbm_kernels_wait_flag(flag_ptr, value, stream)
