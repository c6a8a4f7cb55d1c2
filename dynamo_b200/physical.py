"""ctypes mirror of the reference's host-side transfer API (lib/kvbm-physical), over libkvbm_physical.so.

Names and argument meaning follow the Rust crate so tests read like the reference's own:
  LayoutConfig                    lib/kvbm-physical/src/layout/config.rs:14-56
  StorageKind / BlockDimension    lib/memory/src/lib.rs, layout/config.rs:151-163
  TransferOptions                 transfer/options.rs:27-81
  TransferManager.register_layout / export_metadata / import_metadata / execute_transfer
                                  manager/mod.rs:101,112,130,227
  select_direct_strategy          transfer/strategy.rs:138-210
  validate_block_transfer         transfer/validation.rs:168-225
  TransferCompleteNotification    transfer/context.rs:438-470

All bytes move in native code (CUDA kernels for device storage, the reference's own memcpy strategy for
host<->host); this module only marshals arguments.  Missing native library => exception, never a fallback.
"""
from __future__ import annotations

import ctypes as C
import enum
import dataclasses
from dataclasses import dataclass
from typing import List, Mapping, Optional, Sequence, Union

from . import _lib, kernels


class KvbmError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"[{ErrorCode(code).name if code in ErrorCode._value2member_map_ else code}] {msg}")
        self.code = code
        self.msg = msg


class ErrorCode(enum.IntEnum):
    OK = 0
    ERR = 1
    CONFIG = 2
    RANGE = 3
    LENGTH_MISMATCH = 4
    DUPLICATE_DST = 5
    OVERLAP = 6
    INCOMPATIBLE = 7
    UNSUPPORTED = 8
    CUDA = 9
    HANDLE = 10
    TIMEOUT = 11
    VERSION = 12


class StorageKind(enum.IntEnum):
    System = 0
    Pinned = 1
    Device = 2
    Disk = 3


class BlockDimension(enum.IntEnum):
    BlockIsFirstDim = 0
    BlockIsSecondDim = 1


class TransferStrategy(enum.IntEnum):
    Memcpy = 0
    CudaAsyncH2D = 1
    CudaAsyncD2H = 2
    CudaAsyncD2D = 3
    NixlRead = 4
    NixlWrite = 5
    NixlReadFlipped = 6
    Invalid = 7


class _CConfig(C.Structure):
    _fields_ = [(n, C.c_size_t) for n in ("num_blocks", "num_layers", "outer_dim", "page_size", "inner_dim",
                                          "alignment", "dtype_width_bytes", "num_heads")] + [("allow_fp8", C.c_int)]


class _CPlan(C.Structure):
    _fields_ = [("two_hop", C.c_int), ("first", C.c_int), ("bounce_location", C.c_int), ("second", C.c_int)]


class _CCaps(C.Structure):
    _fields_ = [("allow_gds", C.c_int), ("allow_gpu_rdma", C.c_int)]


class _COptions(C.Structure):
    _fields_ = [
        ("has_layer_range", C.c_int),
        ("layer_begin", C.c_size_t),
        ("layer_end", C.c_size_t),
        ("cuda_stream", C.c_void_p),
        ("use_caller_stream", C.c_int),
        ("cast_mode", C.c_int),
        ("max_ctas", C.c_int),
        ("layer_ready_flags", C.c_void_p),
        ("layer_done_flags", C.c_void_p),
        ("epoch", C.c_uint32),
        ("gate_timeout_ms", C.c_int),
        ("multicast", C.c_int),
        ("done_flag", C.c_void_p),
        ("bounce_layout", C.c_uint64),
        ("bounce_block_ids", C.c_void_p),
        ("num_bounce_blocks", C.c_size_t),
        ("src_kv_layout", C.c_int),
        ("dst_kv_layout", C.c_int),
        ("gate_mode", C.c_int),
        ("per_dst_done_flags", C.c_void_p),
        ("per_dst_layer_done_flags", C.c_void_p),
        ("src_head_begin", C.c_size_t),
        ("dst_head_begin", C.c_size_t),
        ("head_count", C.c_size_t),
        ("cast_scales", C.c_void_p),
        ("num_cast_scales", C.c_size_t),
    ]


class _CHeadWindow(C.Structure):
    _fields_ = [(n, C.c_size_t) for n in ("src_rank", "src_head_begin", "dst_head_begin", "head_count")]


class _CShardWindow(C.Structure):
    _fields_ = [(n, C.c_size_t) for n in ("src_rank", "src_layer_begin", "dst_layer_begin", "layer_count", "src_head_begin",
                                          "dst_head_begin", "head_count")]


class _CScatterWindow(C.Structure):
    _fields_ = [(n, C.c_size_t) for n in ("dst_rank", "src_layer_begin", "dst_layer_begin", "layer_count", "src_head_begin", "dst_head_begin",
                                          "head_count")]


class _CRepageBatchSeq(C.Structure):
    """struct kvbm_repage_batch_seq"""
    _fields_ = [("token_begin", C.c_size_t), ("token_end", C.c_size_t), ("src_ids", C.c_void_p), ("n_src", C.c_size_t),
                ("dst_ids", C.c_void_p), ("n_dst", C.c_size_t)]


class _CRepageRouteSeq(C.Structure):
    """struct kvbm_repage_route_seq"""
    _fields_ = [("token_begin", C.c_size_t), ("token_end", C.c_size_t), ("src_ids", C.c_void_p), ("n_src", C.c_size_t),
                ("dst_ids", C.c_void_p), ("n_dst", C.c_size_t), ("src_mask", C.c_uint32)]


class _CScatterBatchSeq(C.Structure):
    """struct kvbm_scatter_batch_seq"""
    _fields_ = [("token_begin", C.c_size_t), ("token_end", C.c_size_t), ("src_ids", C.c_void_p), ("n_src", C.c_size_t),
                ("dst_ids", C.c_void_p), ("n_dst", C.c_size_t)]


class _CScatterRouteSeq(C.Structure):
    """struct kvbm_scatter_route_seq"""
    _fields_ = [("token_begin", C.c_size_t), ("token_end", C.c_size_t), ("src_ids", C.c_void_p), ("n_src", C.c_size_t),
                ("dst_ids", C.c_void_p), ("n_dst", C.c_size_t), ("dst_mask", C.c_uint32)]


class _CLayerStream(C.Structure):
    """struct kvbm_layer_stream"""
    _fields_ = [("src_layer_ready_flags", C.c_void_p), ("num_srcs", C.c_size_t), ("layer_done_flags", C.c_void_p)]


@dataclass
class LayoutConfig:
    num_blocks: int
    num_layers: int
    outer_dim: int
    page_size: int
    inner_dim: int
    alignment: int = 1
    dtype_width_bytes: int = 2
    num_heads: Optional[int] = None
    allow_fp8: bool = False

    def _c(self) -> _CConfig:
        return _CConfig(self.num_blocks, self.num_layers, self.outer_dim, self.page_size, self.inner_dim,
                        self.alignment, self.dtype_width_bytes, self.num_heads or 0, int(self.allow_fp8))

    def validate(self) -> None:
        _check(lib().kvbm_layout_config_validate(C.byref(self._c())))

    def required_bytes(self) -> int:
        return lib().kvbm_layout_required_bytes(C.byref(self._c()))

    def bytes_per_block(self) -> int:
        return lib().kvbm_layout_bytes_per_block(C.byref(self._c()))

    def region_size(self) -> int:
        return self.page_size * self.inner_dim * self.dtype_width_bytes


@dataclass
class TransferOptions:
    layer_range: Optional[range] = None
    cuda_stream: Optional[int] = None     # raw cudaStream_t; when set the caller manages synchronisation
    cast_mode: int = 0
    max_ctas: int = 0
    layer_ready_flags: int = 0
    layer_done_flags: int = 0
    epoch: int = 0
    gate_timeout_ms: int = 0
    multicast: int = 0                    # destination layout lives in a MulticastGroup.map() range (NVLS)
    done_flag: int = 0                    # word on the destination GPU that receives `epoch` on completion (cf. nixl_write_notification)
    bounce_buffer: Optional[tuple] = None # (layout handle, block ids): BounceBuffer of options.rs:45-51 for two-hop transfers
    src_kv_layout: int = 0                # KvBlockLayout overrides (options.rs:63-80); a pair needing a transform runs the permuting launch
    dst_kv_layout: int = 0
    gate_mode: int = 0                    # kernels.GATE_AUTO / GATE_SPIN / GATE_STREAM_WAIT
    per_dst_done_flags: Optional[Sequence[int]] = None        # fan-out: one done-flag address per destination (0 = none)
    per_dst_layer_done_flags: Optional[Sequence[int]] = None  # fan-out: one layer-done array address per destination
    head_window: Optional[tuple] = None   # (src_head_begin, dst_head_begin, head_count): move only these heads (TP re-shard)
    # fp8 KV-cache scales: a contiguous float32 CUDA tensor of num_layers * outer_dim entries (entry l * outer_dim + o scales the
    # fp8 side of layer l, outer index o), applied by the cast; kept alive by this object
    cast_scales: Optional[object] = None

    @staticmethod
    def from_layer_range(layer_range: Optional[range]) -> "TransferOptions":
        return TransferOptions(layer_range=layer_range)

    def _c(self) -> _COptions:
        lr = self.layer_range
        bl, bids, nb = 0, None, 0
        if self.bounce_buffer is not None:
            bl, ids = self.bounce_buffer
            self._bounce_keepalive = (C.c_size_t * max(1, len(ids)))(*[int(x) for x in ids])
            bids, nb = C.cast(self._bounce_keepalive, C.c_void_p), len(ids)
        sb, db, k = self.head_window if self.head_window is not None else (0, 0, 0)
        return _COptions(int(lr is not None), lr.start if lr is not None else 0, lr.stop if lr is not None else 0,
                         self.cuda_stream or 0, int(self.cuda_stream is not None), int(self.cast_mode), self.max_ctas,
                         self.layer_ready_flags, self.layer_done_flags, self.epoch, self.gate_timeout_ms,
                         int(self.multicast), self.done_flag, int(bl), bids, nb, int(self.src_kv_layout),
                         int(self.dst_kv_layout), int(self.gate_mode), self._ptr_array("_pd", self.per_dst_done_flags),
                         self._ptr_array("_pl", self.per_dst_layer_done_flags), int(sb), int(db), int(k),
                         kernels.scales_ptr(self.cast_scales), self._num_scales())

    def _num_scales(self) -> int:
        s = self.cast_scales
        if s is None:
            return 0
        if isinstance(s, int):
            raise TypeError("TransferOptions.cast_scales takes a float32 tensor (its numel is the scale count), not an address")
        return int(s.numel()) if hasattr(s, "numel") else int(s.size)

    def _ptr_array(self, keep: str, ptrs):
        if ptrs is None:
            return None
        arr = (C.c_void_p * max(1, len(ptrs)))(*[int(p) or None for p in ptrs])
        setattr(self, keep, arr)          # keep the array alive as long as the options object
        return C.cast(arr, C.c_void_p)


@dataclass
class TransferPlan:
    two_hop: bool
    first: TransferStrategy
    bounce_location: Optional[StorageKind] = None
    second: Optional[TransferStrategy] = None


_configured = False

EXPORTED_SYMBOLS = [
    "kvbm_last_error", "kvbm_layout_config_validate", "kvbm_layout_required_bytes", "kvbm_layout_bytes_per_block",
    "kvbm_select_direct_strategy", "kvbm_validate_block_transfer", "kvbm_manager_create", "kvbm_manager_destroy",
    "kvbm_manager_register_fully_contiguous", "kvbm_manager_register_layer_separate", "kvbm_manager_unregister",
    "kvbm_layout_memory_region", "kvbm_layout_is_fully_contiguous", "kvbm_manager_enable_peer_access",
    "kvbm_manager_export_metadata", "kvbm_manager_import_metadata", "kvbm_manager_import_metadata_mapped", "kvbm_manager_execute_transfer",
    "kvbm_manager_execute_fanout", "kvbm_notification_is_complete", "kvbm_notification_wait",
    "kvbm_manager_bytes_moved", "kvbm_manager_h2d_bytes", "kvbm_manager_set_capabilities",
    "kvbm_manager_export_serialized_layout", "kvbm_manager_import_serialized_layout", "kvbm_layout_descriptor_json",
    "kvbm_manager_import_descriptor_json", "kvbm_select_transform_kernel", "kvbm_kv_layout_requires_transform",
    "kvbm_manager_set_kv_block_layout", "kvbm_manager_kv_block_layout",
    "kvbm_select_direct_strategy_remote", "kvbm_select_strategy", "kvbm_manager_select_strategy",
    "kvbm_mc_supported", "kvbm_mc_group_create", "kvbm_mc_group_export_fd", "kvbm_mc_group_import_fd",
    "kvbm_mc_group_size", "kvbm_mc_group_add_device", "kvbm_mc_group_bind_local", "kvbm_mc_group_bind_addr", "kvbm_mc_group_map",
    "kvbm_mc_group_destroy", "kvbm_tp_reshard_plan", "kvbm_manager_execute_gather", "kvbm_manager_execute_repage",
    "kvbm_manager_execute_repage_gather", "kvbm_manager_execute_gather_streamed", "kvbm_manager_execute_repage_gather_streamed",
    "kvbm_tp_pp_reshard_plan", "kvbm_manager_execute_stage_gather", "kvbm_manager_execute_stage_repage_gather",
    "kvbm_manager_execute_repage_batch", "kvbm_tp_pp_scatter_plan", "kvbm_manager_execute_repage_scatter",
    "kvbm_manager_execute_repage_scatter_streamed", "kvbm_manager_execute_repage_scatter_batch",
    "kvbm_manager_execute_repage_scatter_routed", "kvbm_manager_execute_repage_batch_routed", "kvbm_manager_execute_repage_anypage",
    "kvbm_manager_execute_repage_scatter_anypage", "kvbm_manager_execute_repage_scatter_routed_anypage",
    "kvbm_manager_execute_repage_batch_routed_anypage",
]


_LIB: Optional[C.CDLL] = None


def lib() -> C.CDLL:
    global _configured, _LIB
    if _LIB is not None:      # hot path: every transfer goes through here twice
        return _LIB
    kernels.lib()  # dependency (resolved through $ORIGIN rpath as well)
    L = _lib.load(_lib.PHYSICAL_SO)
    if not _configured:
        vp, sz, i, u64 = C.c_void_p, C.c_size_t, C.c_int, C.c_uint64
        P = C.POINTER
        L.kvbm_last_error.restype = C.c_char_p
        L.kvbm_layout_config_validate.argtypes = [P(_CConfig)]
        L.kvbm_layout_required_bytes.argtypes = [P(_CConfig)]
        L.kvbm_layout_required_bytes.restype = sz
        L.kvbm_layout_bytes_per_block.argtypes = [P(_CConfig)]
        L.kvbm_layout_bytes_per_block.restype = sz
        L.kvbm_select_direct_strategy.argtypes = [i, i, P(_CCaps), P(_CPlan)]
        L.kvbm_select_direct_strategy_remote.argtypes = [i, i, i, P(_CCaps), P(_CPlan)]
        L.kvbm_select_strategy.argtypes = [i, i, i, i, P(_CCaps), P(_CPlan)]
        L.kvbm_manager_select_strategy.argtypes = [vp, u64, u64, P(_CPlan)]
        L.kvbm_validate_block_transfer.argtypes = [P(sz), sz, P(sz), sz, sz, sz, i]
        L.kvbm_manager_create.argtypes = [i, u64, P(vp)]
        L.kvbm_manager_destroy.argtypes = [vp]
        L.kvbm_manager_destroy.restype = None
        L.kvbm_manager_register_fully_contiguous.argtypes = [vp, P(_CConfig), vp, sz, i, i, P(u64)]
        L.kvbm_manager_register_layer_separate.argtypes = [vp, P(_CConfig), P(vp), P(sz), i, i, i, P(u64)]
        L.kvbm_manager_unregister.argtypes = [vp, u64]
        L.kvbm_layout_memory_region.argtypes = [vp, u64, sz, sz, sz, P(sz), P(sz)]
        L.kvbm_layout_is_fully_contiguous.argtypes = [vp, u64]
        L.kvbm_manager_enable_peer_access.argtypes = [vp, i]
        L.kvbm_manager_export_metadata.argtypes = [vp, u64, vp, sz, P(sz)]
        L.kvbm_manager_import_metadata.argtypes = [vp, vp, sz, P(u64)]
        L.kvbm_manager_import_metadata_mapped.argtypes = [vp, vp, sz, P(vp), sz, P(u64)]
        # the id lists are `const size_t*`; declared void* so a raw address (numpy buffer) passes without a ctypes cast
        L.kvbm_manager_execute_transfer.argtypes = [vp, u64, vp, u64, vp, sz, P(_COptions), P(u64)]
        L.kvbm_manager_execute_fanout.argtypes = [vp, u64, i, P(u64), P(P(sz)), P(P(sz)), sz, i, P(_COptions), P(u64)]
        L.kvbm_manager_set_capabilities.argtypes = [vp, P(_CCaps)]
        L.kvbm_manager_set_kv_block_layout.argtypes = [vp, u64, i]
        L.kvbm_manager_kv_block_layout.argtypes = [vp, u64]
        L.kvbm_select_transform_kernel.argtypes = [i, i]
        L.kvbm_kv_layout_requires_transform.argtypes = [i, i]
        L.kvbm_tp_reshard_plan.argtypes = [sz, sz, sz, sz, P(_CHeadWindow), sz, P(sz)]
        L.kvbm_manager_execute_gather.argtypes = [vp, sz, P(u64), P(P(sz)), u64, vp, sz, P(_CHeadWindow), sz, P(_COptions), P(u64)]
        L.kvbm_manager_execute_repage.argtypes = [vp, u64, vp, sz, u64, vp, sz, sz, sz, P(_COptions), P(u64)]
        L.kvbm_manager_execute_repage_gather.argtypes = [vp, sz, P(u64), P(P(sz)), sz, u64, vp, sz, sz, sz, P(_CHeadWindow), sz,
                                                         P(_COptions), P(u64)]
        L.kvbm_manager_execute_gather_streamed.argtypes = [vp, sz, P(u64), P(P(sz)), u64, vp, sz, P(_CHeadWindow), sz, P(_CLayerStream),
                                                           P(_COptions), P(u64)]
        L.kvbm_manager_execute_repage_gather_streamed.argtypes = [vp, sz, P(u64), P(P(sz)), sz, u64, vp, sz, sz, sz, P(_CHeadWindow), sz,
                                                                  P(_CLayerStream), P(_COptions), P(u64)]
        L.kvbm_tp_pp_reshard_plan.argtypes = [sz, sz, sz, sz, P(sz), sz, sz, P(sz), sz, P(_CShardWindow), sz, P(sz)]
        L.kvbm_manager_execute_stage_gather.argtypes = [vp, sz, P(u64), P(P(sz)), u64, vp, sz, P(_CShardWindow), sz, P(_CLayerStream),
                                                        P(_COptions), P(u64)]
        L.kvbm_manager_execute_stage_repage_gather.argtypes = [vp, sz, P(u64), P(P(sz)), sz, u64, vp, sz, sz, sz, P(_CShardWindow), sz,
                                                               P(_CLayerStream), P(_COptions), P(u64)]
        L.kvbm_manager_execute_repage_batch.argtypes = [vp, sz, P(u64), u64, P(_CRepageBatchSeq), sz, P(_CShardWindow), sz, P(_CLayerStream),
                                                        P(_COptions), P(u64)]
        L.kvbm_manager_execute_repage_anypage.argtypes = L.kvbm_manager_execute_repage_batch.argtypes
        L.kvbm_manager_execute_repage_batch_routed.argtypes = [vp, sz, P(u64), u64, P(_CRepageRouteSeq), sz, P(_CShardWindow), sz,
                                                               P(_CLayerStream), P(_COptions), P(u64)]
        L.kvbm_manager_execute_repage_batch_routed_anypage.argtypes = L.kvbm_manager_execute_repage_batch_routed.argtypes
        L.kvbm_tp_pp_scatter_plan.argtypes = [sz, sz, sz, sz, P(sz), sz, sz, P(sz), sz, P(_CScatterWindow), sz, P(sz)]
        L.kvbm_manager_execute_repage_scatter.argtypes = [vp, u64, vp, sz, sz, P(u64), P(P(sz)), sz, sz, sz, P(_CScatterWindow), sz,
                                                          P(_COptions), P(u64)]
        L.kvbm_manager_execute_repage_scatter_streamed.argtypes = [vp, u64, vp, sz, sz, P(u64), P(P(sz)), sz, sz, sz, P(_CScatterWindow),
                                                                   sz, P(_CLayerStream), P(_COptions), P(u64)]
        L.kvbm_manager_execute_repage_scatter_batch.argtypes = [vp, u64, sz, P(u64), P(_CScatterBatchSeq), sz, P(_CScatterWindow), sz,
                                                                P(_CLayerStream), P(_COptions), P(u64)]
        L.kvbm_manager_execute_repage_scatter_anypage.argtypes = L.kvbm_manager_execute_repage_scatter_batch.argtypes
        L.kvbm_manager_execute_repage_scatter_routed.argtypes = [vp, u64, sz, P(u64), P(_CScatterRouteSeq), sz, P(_CScatterWindow), sz,
                                                                 P(_CLayerStream), P(_COptions), P(u64)]
        L.kvbm_manager_execute_repage_scatter_routed_anypage.argtypes = L.kvbm_manager_execute_repage_scatter_routed.argtypes
        L.kvbm_notification_is_complete.argtypes = [vp, u64]
        L.kvbm_notification_wait.argtypes = [vp, u64, C.c_int64]
        L.kvbm_manager_bytes_moved.argtypes = [vp]
        L.kvbm_manager_bytes_moved.restype = u64
        L.kvbm_manager_h2d_bytes.argtypes = [vp]
        L.kvbm_manager_h2d_bytes.restype = u64
        L.kvbm_manager_export_serialized_layout.argtypes = [vp, vp, sz, P(sz)]
        L.kvbm_manager_import_serialized_layout.argtypes = [vp, vp, sz, P(u64), sz, P(sz)]
        L.kvbm_layout_descriptor_json.argtypes = [vp, u64, vp, sz, P(sz)]
        L.kvbm_manager_import_descriptor_json.argtypes = [vp, C.c_char_p, sz, P(u64)]
        L.kvbm_mc_supported.argtypes = [i]
        L.kvbm_mc_group_create.argtypes = [i, sz, i, P(vp)]
        L.kvbm_mc_group_export_fd.argtypes = [vp, P(i)]
        L.kvbm_mc_group_import_fd.argtypes = [i, i, sz, P(vp)]
        L.kvbm_mc_group_size.argtypes = [vp]
        L.kvbm_mc_group_size.restype = sz
        L.kvbm_mc_group_add_device.argtypes = [vp, i]
        L.kvbm_mc_group_bind_local.argtypes = [vp, i, P(vp)]
        L.kvbm_mc_group_bind_addr.argtypes = [vp, i, vp, sz]
        L.kvbm_mc_group_map.argtypes = [vp, i, P(vp)]
        L.kvbm_mc_group_destroy.argtypes = [vp]
        L.kvbm_mc_group_destroy.restype = None
        _configured = True
    _LIB = L
    return L


def _check(rc: int) -> None:
    if rc != 0:
        raise KvbmError(rc, lib().kvbm_last_error().decode(errors="replace"))


try:
    import numpy as _np
    _NP_ID_DTYPES = (_np.dtype(_np.uint64), _np.dtype(_np.int64))
except ImportError:  # pragma: no cover
    _np = None
    _NP_ID_DTYPES = ()


def _size_array(ids: Sequence[int]):
    """Host block-id list -> `const size_t*`.  numpy int64/uint64 arrays are passed without copying."""
    n = len(ids)
    if _np is not None and isinstance(ids, _np.ndarray) and ids.dtype in _NP_ID_DTYPES and ids.flags.c_contiguous:
        return _NpView(ids), n
    return (C.c_size_t * max(1, n))(*[int(x) for x in ids]), n


class _NpView:
    """Keeps the numpy array alive and presents its buffer as a pointer argument."""
    __slots__ = ("arr", "addr")

    def __init__(self, arr):
        self.arr = arr
        self.addr = arr.__array_interface__["data"][0]

    @property
    def _as_parameter_(self):     # only the fan-out / validation paths need a typed pointer
        return C.cast(self.addr, C.POINTER(C.c_size_t))


def _plan(plan: _CPlan) -> TransferPlan:
    if plan.two_hop:
        return TransferPlan(True, TransferStrategy(plan.first), StorageKind(plan.bounce_location),
                            TransferStrategy(plan.second))
    return TransferPlan(False, TransferStrategy(plan.first))


def select_direct_strategy(src: StorageKind, dst: StorageKind, allow_gds: bool = False,
                           allow_gpu_rdma: bool = False, dst_is_remote: bool = False) -> TransferPlan:
    """select_direct_strategy(src, dst, dst_is_remote, capabilities) -- transfer/strategy.rs:138-243."""
    plan = _CPlan()
    caps = _CCaps(int(allow_gds), int(allow_gpu_rdma))
    _check(lib().kvbm_select_direct_strategy_remote(int(src), int(dst), int(dst_is_remote), C.byref(caps), C.byref(plan)))
    return _plan(plan)


def select_strategy(src: StorageKind, src_is_local: bool, dst: StorageKind, dst_is_local: bool, allow_gds: bool = False,
                    allow_gpu_rdma: bool = False) -> TransferPlan:
    """select_strategy + select_remote_strategy_v2 -- transfer/strategy.rs:78-108,245-281."""
    plan = _CPlan()
    caps = _CCaps(int(allow_gds), int(allow_gpu_rdma))
    _check(lib().kvbm_select_strategy(int(src), int(src_is_local), int(dst), int(dst_is_local), C.byref(caps), C.byref(plan)))
    return _plan(plan)


class TransformKernel(enum.IntEnum):
    """TransformKernel (transfer/executor/mod.rs:27-41)"""
    NONE = 0
    BlockToUniversal = 1
    UniversalToBlock = 2
    OperationalTranspose = 3
    Unsupported = 4
    UniversalToUniversal = 5   # extension (a TODO in the reference); executed by transfers, never selected by the function below


def select_transform_kernel(src: "kernels.KvBlockLayout", dst: "kernels.KvBlockLayout") -> TransformKernel:
    """select_transform_kernel (transfer/executor/mod.rs:46-100)."""
    return TransformKernel(lib().kvbm_select_transform_kernel(int(src), int(dst)))


def requires_transform(a: "kernels.KvBlockLayout", b: "kernels.KvBlockLayout") -> bool:
    """KvBlockLayout::requires_transform (layout/kv_block_layout.rs:107-119)."""
    return bool(lib().kvbm_kv_layout_requires_transform(int(a), int(b)))


def validate_block_transfer(src_ids: Sequence[int], dst_ids: Sequence[int], src_num_blocks: int,
                            dst_num_blocks: int, same_layout: bool = False) -> None:
    s, ns = _size_array(src_ids)
    d, nd = _size_array(dst_ids)
    _check(lib().kvbm_validate_block_transfer(s, ns, d, nd, src_num_blocks, dst_num_blocks, int(same_layout)))


@dataclass(frozen=True)
class HeadWindow:
    """One entry of a TP re-shard plan: heads [src_head_begin, +head_count) of source rank src_rank's blocks are heads
    [dst_head_begin, +head_count) of the decode rank's blocks (rank-local indices)."""
    src_rank: int
    src_head_begin: int
    dst_head_begin: int
    head_count: int


def tp_reshard_plan(num_kv_heads: int, src_tp: int, dst_tp: int, dst_rank: int) -> List[HeadWindow]:
    """Which source rank supplies which heads of decode rank `dst_rank` (kvbm_tp_reshard_plan, include/kvbm_physical.h): vLLM's
    head ownership on both sides, replica dst_rank % replicas of a replicated source head, ascending destination heads, adjacent
    heads of one source merged."""
    n = C.c_size_t()
    _check(lib().kvbm_tp_reshard_plan(num_kv_heads, src_tp, dst_tp, dst_rank, None, 0, C.byref(n)))
    out = (_CHeadWindow * max(1, n.value))()
    _check(lib().kvbm_tp_reshard_plan(num_kv_heads, src_tp, dst_tp, dst_rank, out, n.value, C.byref(n)))
    return [HeadWindow(w.src_rank, w.src_head_begin, w.dst_head_begin, w.head_count) for w in out[:n.value]]


@dataclass(frozen=True)
class ShardWindow:
    """One entry of a PP x TP re-shard plan: heads [src_head_begin, +head_count) of layers [src_layer_begin, +layer_count) of
    source rank src_rank's blocks are heads [dst_head_begin, +head_count) of layers [dst_layer_begin, +layer_count) of the decode
    rank's blocks.  Layers are stage-local on each side (a pool's layer 0 is its stage's first layer), heads rank-local."""
    src_rank: int
    src_layer_begin: int
    dst_layer_begin: int
    layer_count: int
    src_head_begin: int
    dst_head_begin: int
    head_count: int


def tp_pp_reshard_plan(num_kv_heads: int, num_layers: int, src_tp: int, src_pp: int, dst_tp: int, dst_pp: int, dst_rank: int,
                       src_stage_layers: Optional[Sequence[int]] = None,
                       dst_stage_layers: Optional[Sequence[int]] = None) -> List[ShardWindow]:
    """Which source rank supplies which layers and heads of decode rank `dst_rank` (kvbm_tp_pp_reshard_plan,
    include/kvbm_physical.h): ranks are pp_rank * tp + tp_rank on both sides; `*_stage_layers` are each stage's layer counts
    (None: an even split, which needs num_layers % pp == 0); for each source stage that shares layers with the decode rank's
    stage, `tp_reshard_plan`'s head windows over the shared layers, in ascending destination layer, then head order."""
    def parts(v):
        return None if v is None else (C.c_size_t * max(1, len(v)))(*[int(x) for x in v])
    sp, dp = parts(src_stage_layers), parts(dst_stage_layers)
    for v, pp in ((src_stage_layers, src_pp), (dst_stage_layers, dst_pp)):
        if v is not None and len(v) != pp:
            raise ValueError(f"{len(v)} stage layer counts for PP {pp}")
    n = C.c_size_t()
    args = (num_kv_heads, num_layers, src_tp, src_pp, sp, dst_tp, dst_pp, dp, dst_rank)
    _check(lib().kvbm_tp_pp_reshard_plan(*args, None, 0, C.byref(n)))
    out = (_CShardWindow * max(1, n.value))()
    _check(lib().kvbm_tp_pp_reshard_plan(*args, out, n.value, C.byref(n)))
    return [ShardWindow(w.src_rank, w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin, w.dst_head_begin, w.head_count)
            for w in out[:n.value]]


@dataclass(frozen=True)
class ScatterWindow:
    """One entry of a scatter plan: heads [src_head_begin, +head_count) of layers [src_layer_begin, +layer_count) of the prefill
    rank's blocks are heads [dst_head_begin, +head_count) of layers [dst_layer_begin, +layer_count) of decode rank dst_rank's blocks
    (stage-local layers, rank-local heads)."""
    dst_rank: int
    src_layer_begin: int
    dst_layer_begin: int
    layer_count: int
    src_head_begin: int
    dst_head_begin: int
    head_count: int


def tp_pp_scatter_plan(num_kv_heads: int, num_layers: int, src_tp: int, src_pp: int, dst_tp: int, dst_pp: int, src_rank: int,
                       src_stage_layers: Optional[Sequence[int]] = None,
                       dst_stage_layers: Optional[Sequence[int]] = None) -> List[ScatterWindow]:
    """Which layers and heads of prefill rank `src_rank` go to which decode rank (kvbm_tp_pp_scatter_plan, include/kvbm_physical.h):
    the windows of `tp_pp_reshard_plan` over every decode rank that read `src_rank`, tagged with their decode rank, in ascending
    (dst_rank, destination layer, destination head) order, so the push and pull plans of one group move the same bytes."""
    def parts(v):
        return None if v is None else (C.c_size_t * max(1, len(v)))(*[int(x) for x in v])
    sp, dp = parts(src_stage_layers), parts(dst_stage_layers)
    for v, pp in ((src_stage_layers, src_pp), (dst_stage_layers, dst_pp)):
        if v is not None and len(v) != pp:
            raise ValueError(f"{len(v)} stage layer counts for PP {pp}")
    n = C.c_size_t()
    args = (num_kv_heads, num_layers, src_tp, src_pp, sp, dst_tp, dst_pp, dp, src_rank)
    _check(lib().kvbm_tp_pp_scatter_plan(*args, None, 0, C.byref(n)))
    out = (_CScatterWindow * max(1, n.value))()
    _check(lib().kvbm_tp_pp_scatter_plan(*args, out, n.value, C.byref(n)))
    return [ScatterWindow(w.dst_rank, w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin, w.dst_head_begin, w.head_count)
            for w in out[:n.value]]


def tile_scatter_plan(plan: Sequence[ScatterWindow], num_workers: int, ranks_per_worker: int) -> List[ScatterWindow]:
    """One decode group's scatter plan (`tp_pp_scatter_plan`) repeated over `num_workers` identical decode workers of
    `ranks_per_worker` ranks each: worker w's copy of a window names destination rank dst_rank + w * ranks_per_worker, so the
    destinations are worker-major and a routed sequence for worker w sets bits w * ranks_per_worker .. +ranks_per_worker - 1."""
    if num_workers < 1 or any(w.dst_rank >= ranks_per_worker for w in plan):
        raise ValueError(f"a plan for {ranks_per_worker} ranks per worker cannot be tiled {num_workers} times")
    return [dataclasses.replace(w, dst_rank=w.dst_rank + k * ranks_per_worker) for k in range(num_workers) for w in plan]


def tile_reshard_plan(plan: Sequence[ShardWindow], num_workers: int, ranks_per_worker: int) -> List[ShardWindow]:
    """One prefill group's re-shard plan (`tp_pp_reshard_plan`) repeated over `num_workers` identical prefill workers of
    `ranks_per_worker` ranks each, the mirror of `tile_scatter_plan`: worker w's copy of a window reads source rank src_rank +
    w * ranks_per_worker, so the sources are worker-major and a routed sequence served by worker w sets bits w * ranks_per_worker
    .. +ranks_per_worker - 1.  The copies of two workers write the same destination heads, which a routed gather allows as long
    as no sequence is routed to both."""
    if num_workers < 1 or any(w.src_rank >= ranks_per_worker for w in plan):
        raise ValueError(f"a plan for {ranks_per_worker} ranks per worker cannot be tiled {num_workers} times")
    return [dataclasses.replace(w, src_rank=w.src_rank + k * ranks_per_worker) for k in range(num_workers) for w in plan]


class TransferCompleteNotification:
    def __init__(self, mgr: "TransferManager", token: int):
        self._mgr, self.token = mgr, token

    def is_complete(self) -> bool:
        rc = lib().kvbm_notification_is_complete(self._mgr._h, self.token)
        if rc == -2:
            raise KvbmError(ErrorCode.TIMEOUT, "gated transfer aborted: a layer_ready flag was not released within the gate timeout")
        if rc < 0:
            raise KvbmError(ErrorCode.HANDLE, "unknown notification")
        return rc == 1

    def wait(self, timeout_s: Optional[float] = 30.0) -> None:
        us = -1 if timeout_s is None else int(timeout_s * 1e6)
        _check(lib().kvbm_notification_wait(self._mgr._h, self.token, us))


class TransferManager:
    """TransferManager over one CUDA device (device < 0: host-only, Memcpy strategy only)."""

    def __init__(self, device: int = 0, worker_id: int = 0):
        h = C.c_void_p()
        _check(lib().kvbm_manager_create(device, worker_id, C.byref(h)))
        self._h = h
        self.device = device

    def close(self) -> None:
        if self._h:
            lib().kvbm_manager_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- layouts ------------------------------------------------------------------------------------
    def register_fully_contiguous(self, config: LayoutConfig, base: int, size: int, storage: StorageKind,
                                  device_id: int = 0) -> int:
        out = C.c_uint64()
        _check(lib().kvbm_manager_register_fully_contiguous(self._h, C.byref(config._c()), base, size, int(storage),
                                                            device_id, C.byref(out)))
        return out.value

    def register_layer_separate(self, config: LayoutConfig, layer_bases: Sequence[int], layer_sizes: Sequence[int],
                                block_dim: BlockDimension, storage: StorageKind, device_id: int = 0) -> int:
        n = len(layer_bases)
        if n != config.num_layers or len(layer_sizes) != n:
            raise KvbmError(ErrorCode.CONFIG, f"Memory region count ({n}) must match num_layers ({config.num_layers})")
        bases = (C.c_void_p * max(1, n))(*[int(b) for b in layer_bases])
        sizes = (C.c_size_t * max(1, n))(*[int(s) for s in layer_sizes])
        out = C.c_uint64()
        _check(lib().kvbm_manager_register_layer_separate(self._h, C.byref(config._c()), bases, sizes, int(block_dim),
                                                          int(storage), device_id, C.byref(out)))
        return out.value

    def unregister(self, handle: int) -> None:
        _check(lib().kvbm_manager_unregister(self._h, handle))

    def memory_region(self, handle: int, block: int, layer: int, outer: int) -> tuple[int, int]:
        a, s = C.c_size_t(), C.c_size_t()
        _check(lib().kvbm_layout_memory_region(self._h, handle, block, layer, outer, C.byref(a), C.byref(s)))
        return a.value, s.value

    def is_fully_contiguous(self, handle: int) -> bool:
        rc = lib().kvbm_layout_is_fully_contiguous(self._h, handle)
        if rc < 0:
            raise KvbmError(ErrorCode.HANDLE, "invalid handle")
        return bool(rc)

    def select_strategy(self, src: int, dst: int) -> TransferPlan:
        """The plan select_strategy (strategy.rs:78-108) gives for two of this manager's layouts."""
        plan = _CPlan()
        _check(lib().kvbm_manager_select_strategy(self._h, src, dst, C.byref(plan)))
        return _plan(plan)

    def set_kv_block_layout(self, handle: int, kv_layout: "kernels.KvBlockLayout") -> None:
        """The format of one block of this layout (builder `.kv_block_layout()` / `.inner_shape()` in the reference).  A transfer
        between layouts whose formats differ is executed as ONE permuting launch (the reference rejects it)."""
        _check(lib().kvbm_manager_set_kv_block_layout(self._h, handle, int(kv_layout)))

    def kv_block_layout(self, handle: int) -> "kernels.KvBlockLayout":
        rc = lib().kvbm_manager_kv_block_layout(self._h, handle)
        if rc < 0:
            raise KvbmError(ErrorCode.HANDLE, "invalid handle")
        return kernels.KvBlockLayout(rc)

    def enable_peer_access(self, peer_device: int) -> None:
        _check(lib().kvbm_manager_enable_peer_access(self._h, peer_device))

    def export_metadata(self, handle: int) -> bytes:
        n = C.c_size_t()
        _check(lib().kvbm_manager_export_metadata(self._h, handle, None, 0, C.byref(n)))
        buf = C.create_string_buffer(n.value)
        _check(lib().kvbm_manager_export_metadata(self._h, handle, buf, n.value, C.byref(n)))
        return buf.raw[:n.value]

    def import_metadata(self, blob: bytes, local_bases: Optional[Sequence[int]] = None) -> int:
        """`local_bases`: this process's own mappings of another process's HOST pool (shared memory), one address per
        allocation; without it a foreign host pool is imported as a descriptor only."""
        out = C.c_uint64()
        buf = C.create_string_buffer(blob, len(blob))
        if local_bases is None:
            _check(lib().kvbm_manager_import_metadata(self._h, buf, len(blob), C.byref(out)))
        else:
            arr = (C.c_void_p * max(1, len(local_bases)))(*[int(b) for b in local_bases])
            _check(lib().kvbm_manager_import_metadata_mapped(self._h, buf, len(blob), arr, len(local_bases), C.byref(out)))
        return out.value

    # -- the reference's wire formats (SURVEY.md 8 f3) ----------------------------------------------
    def export_serialized_layout(self) -> bytes:
        """`TransferManager::export_metadata()` (manager/mod.rs:112): every local host/device layout in ONE
        `SerializedLayout` blob (bincode 2 over `RdmaLayoutDescriptors`, manager/metadata.rs:87-134)."""
        n = C.c_size_t()
        _check(lib().kvbm_manager_export_serialized_layout(self._h, None, 0, C.byref(n)))
        buf = C.create_string_buffer(max(1, n.value))
        _check(lib().kvbm_manager_export_serialized_layout(self._h, buf, n.value, C.byref(n)))
        return buf.raw[:n.value]

    def import_serialized_layout(self, blob: bytes) -> List[int]:
        """`TransferManager::import_metadata()` (manager/mod.rs:130): handles of the imported remote layouts."""
        buf = C.create_string_buffer(blob, len(blob))
        n = C.c_size_t()
        _check(lib().kvbm_manager_import_serialized_layout(self._h, buf, len(blob), None, 0, C.byref(n)))
        out = (C.c_uint64 * max(1, n.value))()
        _check(lib().kvbm_manager_import_serialized_layout(self._h, buf, len(blob), out, n.value, C.byref(n)))
        return [int(out[i]) for i in range(n.value)]

    def layout_descriptor_json(self, handle: int) -> str:
        """`LayoutDescriptor::to_json` (layout/serialize.rs:96-103) of a registered layout."""
        n = C.c_size_t()
        _check(lib().kvbm_layout_descriptor_json(self._h, handle, None, 0, C.byref(n)))
        buf = C.create_string_buffer(max(1, n.value))
        _check(lib().kvbm_layout_descriptor_json(self._h, handle, buf, n.value, C.byref(n)))
        return buf.raw[:n.value].decode()

    def import_descriptor_json(self, text: str) -> int:
        """`LayoutDescriptor::from_json` + `PhysicalLayout::from_descriptor` (layout/physical.rs:203-262)."""
        raw = text.encode()
        out = C.c_uint64()
        _check(lib().kvbm_manager_import_descriptor_json(self._h, raw, len(raw), C.byref(out)))
        return out.value

    # -- transfers ----------------------------------------------------------------------------------
    def execute_transfer(self, src: int, src_block_ids: Sequence[int], dst: int, dst_block_ids: Sequence[int],
                         options: Optional[TransferOptions] = None) -> TransferCompleteNotification:
        if len(src_block_ids) != len(dst_block_ids):
            # executor/memcpy.rs:38-44: length mismatch is rejected before anything else
            raise KvbmError(ErrorCode.LENGTH_MISMATCH,
                            f"Block ID lists have mismatched lengths: src={len(src_block_ids)}, dst={len(dst_block_ids)}, bounce=None")
        s, n = _size_array(src_block_ids)
        d, _ = _size_array(dst_block_ids)
        tok = C.c_uint64()
        o = options._c() if options is not None else _COptions()
        rc = lib().kvbm_manager_execute_transfer(self._h, src, s.addr if type(s) is _NpView else s, dst,
                                                 d.addr if type(d) is _NpView else d, n, C.byref(o), C.byref(tok))
        if rc:
            _check(rc)
        return TransferCompleteNotification(self, tok.value)

    def execute_reshard(self, sources: Mapping[int, tuple], dst: int, dst_block_ids: Sequence[int], plan: Sequence[HeadWindow],
                        options: Union[None, TransferOptions, Sequence[TransferOptions]] = None) -> List[TransferCompleteNotification]:
        """Assemble blocks of a decode rank from the source ranks' blocks, one `execute_transfer` with a head window per plan entry
        (`tp_reshard_plan`).  `sources` maps a source rank to (layout handle, block ids); `dst_block_ids[i]` receives head
        windows of each source's block i.  The windows of one destination block are byte-disjoint, so the transfers may run on
        different manager streams at once.  `options` is applied to every entry, or is one TransferOptions per entry -- the way to
        give each entry its own done_flag (there is no combined flag).  Returns one notification per entry.  `execute_gather`
        runs the same plan as one launch with one notification and one done_flag."""
        per = list(options) if isinstance(options, (list, tuple)) else [options] * len(plan)
        if len(per) != len(plan):
            raise ValueError(f"{len(per)} options for {len(plan)} plan entries")
        if len(plan) > 1 and not isinstance(options, (list, tuple)) and options is not None and options.done_flag:
            raise ValueError("one done_flag would be written by every entry of the plan: pass one TransferOptions per entry")
        notes = []
        for w, o in zip(plan, per):
            h, ids = sources[w.src_rank]
            o = dataclasses.replace(o or TransferOptions(), head_window=(w.src_head_begin, w.dst_head_begin, w.head_count))
            notes.append(self.execute_transfer(h, ids, dst, dst_block_ids, o))
        return notes

    @staticmethod
    def _gather_args(sources: Mapping[int, tuple], ranks: Sequence[int], dst_block_ids: Sequence[int], plan: Sequence[HeadWindow]):
        """The C arguments of a gather: the plan's source ranks in `ranks` order (the C sources), their handles and id lists, the
        destination's ids and count, the windows with src_rank as an index into `ranks`.  The id arrays are returned so that they
        outlive the call."""
        index = {r: i for i, r in enumerate(ranks)}
        hs = (C.c_uint64 * max(1, len(ranks)))(*[sources[r][0] for r in ranks])
        s_arrays = [_size_array(sources[r][1])[0] for r in ranks]
        d, nd = _size_array(dst_block_ids)
        PP = C.POINTER(C.c_size_t)
        as_ptr = lambda a: a._as_parameter_ if isinstance(a, _NpView) else C.cast(a, PP)  # noqa: E731
        sp = (PP * max(1, len(ranks)))(*[as_ptr(a) for a in s_arrays])
        ws = (_CHeadWindow * max(1, len(plan)))(*[_CHeadWindow(index[w.src_rank], w.src_head_begin, w.dst_head_begin, w.head_count)
                                                  for w in plan])
        return hs, s_arrays, sp, d.addr if type(d) is _NpView else d, nd, ws

    def _gather_call(self, sources: Mapping[int, tuple], dst_block_ids: Sequence[int], plan: Sequence[HeadWindow]):
        """`execute_gather`'s source ranks, after its id-count check, and `_gather_args`."""
        ranks = sorted({w.src_rank for w in plan})
        n = len(dst_block_ids)
        if any(len(sources[r][1]) != n for r in ranks):
            raise KvbmError(ErrorCode.LENGTH_MISMATCH, "Block ID lists have mismatched lengths")
        return ranks, self._gather_args(sources, ranks, dst_block_ids, plan)

    def _repage_gather_call(self, sources: Mapping[int, tuple], dst_block_ids: Sequence[int], plan: Sequence[HeadWindow], tokens: range):
        """`execute_repage_gather`'s source ranks and source id count, after its range and id-count checks, and `_gather_args`."""
        if tokens.step != 1:
            raise ValueError("tokens must be a range with step 1")
        ranks = sorted({w.src_rank for w in plan})
        n_src = len(sources[ranks[0]][1]) if ranks else 0
        if any(len(sources[r][1]) != n_src for r in ranks):
            raise KvbmError(ErrorCode.LENGTH_MISMATCH, "the sources' block id lists have different lengths")
        return ranks, n_src, self._gather_args(sources, ranks, dst_block_ids, plan)

    @staticmethod
    def _shard_windows(ranks: Sequence[int], plan: Sequence[ShardWindow]):
        """The C windows of a staged plan, with src_rank as an index into `ranks`."""
        index = {r: i for i, r in enumerate(ranks)}
        return (_CShardWindow * max(1, len(plan)))(*[_CShardWindow(index[w.src_rank], w.src_layer_begin, w.dst_layer_begin, w.layer_count,
                                                                   w.src_head_begin, w.dst_head_begin, w.head_count) for w in plan])

    @staticmethod
    def _layer_stream(ranks: Sequence[int], ready_flags: Mapping[int, int], layer_done_flags: int) -> "_CLayerStream":
        """struct kvbm_layer_stream for the plan's source ranks; a rank missing from `ready_flags` passes NULL (rejected)."""
        flags = (C.c_void_p * max(1, len(ranks)))(*[int(ready_flags.get(r, 0)) or None for r in ranks])
        ls = _CLayerStream(C.cast(flags, C.c_void_p), len(ranks), layer_done_flags or None)
        ls._keep = flags
        return ls

    def execute_gather(self, sources: Mapping[int, tuple], dst: int, dst_block_ids: Sequence[int], plan: Sequence[HeadWindow],
                       options: Optional[TransferOptions] = None) -> TransferCompleteNotification:
        """`execute_reshard` as ONE hand-off (kvbm_manager_execute_gather): the same `sources` mapping (source rank -> (layout
        handle, block ids)) and plan, at most 16 windows, moved by one permuting launch.  Returns one notification, and
        `options.done_flag` is written once, after every window's bytes landed.  `options.head_window` must be None."""
        ranks, (hs, _keep, sp, d, n, ws) = self._gather_call(sources, dst_block_ids, plan)
        tok = C.c_uint64()
        o = (options or TransferOptions())._c()
        _check(lib().kvbm_manager_execute_gather(self._h, len(ranks), hs, sp, dst, d, n, ws, len(plan), C.byref(o), C.byref(tok)))
        return TransferCompleteNotification(self, tok.value)

    def execute_gather_streamed(self, sources: Mapping[int, tuple], dst: int, dst_block_ids: Sequence[int], plan: Sequence[HeadWindow],
                                ready_flags: Mapping[int, int], options: Optional[TransferOptions] = None,
                                layer_done_flags: int = 0) -> TransferCompleteNotification:
        """`execute_gather` streamed layer by layer (kvbm_manager_execute_gather_streamed): `ready_flags` maps a source rank to
        the address of its [num_layers] u32 ready flags, and layer l of that source is read only after its flag l has reached
        `options.epoch`; `layer_done_flags` (an address on the destination, or 0) gets entry l = epoch once layer l of every
        window landed.  A one-window plan streams a plain format change (a window over every head of both sides) or a single
        re-shard window.  Options: those of `execute_gather`, plus epoch, gate_mode, gate_timeout_ms, max_ctas and done_flag; the
        options' own layer flags stay rejected.  The bytes and bytes_moved are `execute_gather`'s."""
        ranks, (hs, _keep, sp, d, n, ws) = self._gather_call(sources, dst_block_ids, plan)
        ls = self._layer_stream(ranks, ready_flags, layer_done_flags)
        tok = C.c_uint64()
        o = (options or TransferOptions())._c()
        _check(lib().kvbm_manager_execute_gather_streamed(self._h, len(ranks), hs, sp, dst, d, n, ws, len(plan), C.byref(ls), C.byref(o),
                                                          C.byref(tok)))
        return TransferCompleteNotification(self, tok.value)

    def execute_stage_gather(self, sources: Mapping[int, tuple], dst: int, dst_block_ids: Sequence[int], plan: Sequence[ShardWindow],
                             options: Optional[TransferOptions] = None, ready_flags: Optional[Mapping[int, int]] = None,
                             layer_done_flags: int = 0) -> TransferCompleteNotification:
        """A PP x TP re-shard's assembly as ONE hand-off (kvbm_manager_execute_stage_gather): `execute_gather` with a layer window
        per plan entry (`tp_pp_reshard_plan`), each source pool holding only its stage's layers.  `sources` maps a source rank to
        (layout handle, block ids), as `execute_gather`.  The options' layer range and cast scales count destination layers.
        `ready_flags` (None: not streamed) maps a source rank to the address of the u32 ready flags over ITS OWN layers, as
        `execute_gather_streamed`; a destination layer waits only for its stage's sources.  `layer_done_flags`: the destination's."""
        ranks, (hs, _keep, sp, d, n, _ws) = self._gather_call(sources, dst_block_ids, plan)
        ws = self._shard_windows(ranks, plan)
        ls = self._layer_stream(ranks, ready_flags, layer_done_flags) if ready_flags is not None else None
        tok = C.c_uint64()
        o = (options or TransferOptions())._c()
        _check(lib().kvbm_manager_execute_stage_gather(self._h, len(ranks), hs, sp, dst, d, n, ws, len(plan),
                                                       C.byref(ls) if ls is not None else None, C.byref(o), C.byref(tok)))
        return TransferCompleteNotification(self, tok.value)

    def execute_repage(self, src: int, src_block_ids: Sequence[int], dst: int, dst_block_ids: Sequence[int], tokens: range,
                       options: Optional[TransferOptions] = None) -> TransferCompleteNotification:
        """Move tokens `tokens` (a step-1 range of sequence positions) between two layouts with different page sizes (one divides
        the other), re-ordering formats and casting as `execute_transfer` would (kvbm_manager_execute_repage).  `src_block_ids` is
        the source table's entries tokens.start // Ps .. ceil(tokens.stop / Ps), `dst_block_ids` the destination's for Pd; every
        destination byte outside the range keeps its value, so a prefix the decode side already holds, or a partial last block,
        is left alone.  Options: layer_range, cast_mode, cast_scales, src_kv_layout / dst_kv_layout, done_flag / epoch and
        cuda_stream; the others are rejected."""
        if tokens.step != 1:
            raise ValueError("tokens must be a range with step 1")
        s, ns = _size_array(src_block_ids)
        d, nd = _size_array(dst_block_ids)
        tok = C.c_uint64()
        o = (options or TransferOptions())._c()
        _check(lib().kvbm_manager_execute_repage(self._h, src, s.addr if type(s) is _NpView else s, ns, dst,
                                                 d.addr if type(d) is _NpView else d, nd, tokens.start, tokens.stop, C.byref(o),
                                                 C.byref(tok)))
        return TransferCompleteNotification(self, tok.value)

    def execute_repage_gather(self, sources: Mapping[int, tuple], dst: int, dst_block_ids: Sequence[int], plan: Sequence[HeadWindow],
                              tokens: range, options: Optional[TransferOptions] = None) -> TransferCompleteNotification:
        """`execute_gather` across engines with different page sizes, as ONE hand-off (kvbm_manager_execute_repage_gather): the
        same `sources` mapping (source rank -> (layout handle, block ids)) and plan, over `execute_repage`'s `tokens` range.  Every
        source has one page size Ps and its ids are its table's entries tokens.start // Ps .. ceil(tokens.stop / Ps);
        `dst_block_ids` are the destination's for its own page.  Options: those of `execute_repage`."""
        ranks, n_src, (hs, _keep, sp, d, n_dst, ws) = self._repage_gather_call(sources, dst_block_ids, plan, tokens)
        tok = C.c_uint64()
        o = (options or TransferOptions())._c()
        _check(lib().kvbm_manager_execute_repage_gather(self._h, len(ranks), hs, sp, n_src, dst, d, n_dst, tokens.start, tokens.stop, ws,
                                                        len(plan), C.byref(o), C.byref(tok)))
        return TransferCompleteNotification(self, tok.value)

    def execute_repage_gather_streamed(self, sources: Mapping[int, tuple], dst: int, dst_block_ids: Sequence[int],
                                       plan: Sequence[HeadWindow], tokens: range, ready_flags: Mapping[int, int],
                                       options: Optional[TransferOptions] = None, layer_done_flags: int = 0) -> TransferCompleteNotification:
        """`execute_repage_gather` streamed layer by layer (kvbm_manager_execute_repage_gather_streamed), with the flags of
        `execute_gather_streamed`.  A one-window plan over every head of both sides streams a plain re-page."""
        ranks, n_src, (hs, _keep, sp, d, n_dst, ws) = self._repage_gather_call(sources, dst_block_ids, plan, tokens)
        ls = self._layer_stream(ranks, ready_flags, layer_done_flags)
        tok = C.c_uint64()
        o = (options or TransferOptions())._c()
        _check(lib().kvbm_manager_execute_repage_gather_streamed(self._h, len(ranks), hs, sp, n_src, dst, d, n_dst, tokens.start,
                                                                 tokens.stop, ws, len(plan), C.byref(ls), C.byref(o), C.byref(tok)))
        return TransferCompleteNotification(self, tok.value)

    def execute_stage_repage_gather(self, sources: Mapping[int, tuple], dst: int, dst_block_ids: Sequence[int], plan: Sequence[ShardWindow],
                                    tokens: range, options: Optional[TransferOptions] = None, ready_flags: Optional[Mapping[int, int]] = None,
                                    layer_done_flags: int = 0) -> TransferCompleteNotification:
        """A PP x TP re-shard's assembly across engines with different page sizes, as ONE hand-off
        (kvbm_manager_execute_stage_repage_gather): `execute_stage_gather`'s plan (`tp_pp_reshard_plan`) over `execute_repage_gather`'s
        `tokens` range.  Every source has one page size Ps and its ids are its table's entries tokens.start // Ps ..
        ceil(tokens.stop / Ps); `dst_block_ids` are the destination's for its own page.  The options' layer range and cast scales
        count destination layers.  `ready_flags` / `layer_done_flags`: as `execute_stage_gather`'s (None: not streamed)."""
        ranks, n_src, (hs, _keep, sp, d, n_dst, _ws) = self._repage_gather_call(sources, dst_block_ids, plan, tokens)
        ws = self._shard_windows(ranks, plan)
        ls = self._layer_stream(ranks, ready_flags, layer_done_flags) if ready_flags is not None else None
        tok = C.c_uint64()
        o = (options or TransferOptions())._c()
        _check(lib().kvbm_manager_execute_stage_repage_gather(self._h, len(ranks), hs, sp, n_src, dst, d, n_dst, tokens.start, tokens.stop,
                                                              ws, len(plan), C.byref(ls) if ls is not None else None, C.byref(o),
                                                              C.byref(tok)))
        return TransferCompleteNotification(self, tok.value)

    def execute_repage_batch(self, sources: Mapping[int, int], dst: int, seqs: Sequence[tuple], plan: Sequence, options: Optional[TransferOptions] = None,
                             ready_flags: Optional[Mapping[int, int]] = None, layer_done_flags: int = 0,
                             num_layers: Optional[int] = None) -> TransferCompleteNotification:
        """A batch of sequences as ONE hand-off (kvbm_manager_execute_repage_batch): what a continuous-batching decode step admits at
        once, each sequence with its own prefix-cache hit, length and block tables.  `sources` maps a source rank to its layout
        handle; `seqs` is a list of (tokens, {src_rank: src_block_ids}, dst_block_ids), each what `execute_stage_repage_gather`
        takes for one request; `plan` is a ShardWindow list, or a HeadWindow list (a PP1 plan) with `num_layers` the destination's
        layer count.  One staged copy of every table, one launch, one notification, `options.done_flag` written once; with
        `ready_flags`, `layer_done_flags[l]` is written once layer l of every sequence landed.  Two sequences may share source
        blocks; a destination block may appear once in the whole batch.  The first rejected sequence raises what
        `execute_stage_repage_gather` would raise for it."""
        return self._repage_batch(lib().kvbm_manager_execute_repage_batch, sources, dst, seqs, plan, options, ready_flags, layer_done_flags,
                                  num_layers)

    def execute_repage_anypage(self, sources: Mapping[int, int], dst: int, seqs: Sequence[tuple], plan: Sequence,
                               options: Optional[TransferOptions] = None, ready_flags: Optional[Mapping[int, int]] = None,
                               layer_done_flags: int = 0, num_layers: Optional[int] = None) -> TransferCompleteNotification:
        """`execute_repage_batch` between engines whose page sizes need not divide each other (kvbm_manager_execute_repage_anypage),
        e.g. a hybrid model's 544-token attention block into 64-token decode pages, or 24 into 16: the same arguments, plan forms,
        errors and streaming.  Pages past the exactness bound (big + small - gcd) * small < 2^32 raise UNSUPPORTED.  With
        dividing pages the destination bytes are `execute_repage_batch`'s."""
        return self._repage_batch(lib().kvbm_manager_execute_repage_anypage, sources, dst, seqs, plan, options, ready_flags,
                                  layer_done_flags, num_layers)

    def _repage_batch(self, entry, sources, dst, seqs, plan, options, ready_flags, layer_done_flags, num_layers):
        """The body of `execute_repage_batch` and `execute_repage_anypage`: `entry` is the C entry they call."""
        if plan and isinstance(plan[0], HeadWindow):
            if num_layers is None:
                raise ValueError("a HeadWindow plan needs num_layers, the destination's layer count")
            plan = [ShardWindow(w.src_rank, 0, 0, num_layers, w.src_head_begin, w.dst_head_begin, w.head_count) for w in plan]
        ranks = sorted({w.src_rank for w in plan})
        hs = (C.c_uint64 * max(1, len(ranks)))(*[sources[r] for r in ranks])
        ws = self._shard_windows(ranks, plan)
        PP = C.POINTER(C.c_size_t)
        keep, cs = [], (_CRepageBatchSeq * max(1, len(seqs)))()
        for c, (tokens, src_ids, dst_ids) in zip(cs, seqs):
            if tokens.step != 1:
                raise ValueError("tokens must be a range with step 1")
            n_src = len(src_ids[ranks[0]]) if ranks else 0
            if any(len(src_ids[r]) != n_src for r in ranks):
                raise KvbmError(ErrorCode.LENGTH_MISMATCH, "the sources' block id lists have different lengths")
            arrays = [_size_array(src_ids[r])[0] for r in ranks]
            d, n_dst = _size_array(dst_ids)
            sp = (C.c_void_p * max(1, len(ranks)))(*[a.addr if type(a) is _NpView else C.addressof(a) for a in arrays])
            keep += [arrays, d, sp]
            c.token_begin, c.token_end, c.src_ids, c.n_src = tokens.start, tokens.stop, C.addressof(sp), n_src
            c.dst_ids, c.n_dst = (d.addr if type(d) is _NpView else C.addressof(d)), n_dst
        ls = self._layer_stream(ranks, ready_flags, layer_done_flags) if ready_flags is not None else None
        tok = C.c_uint64()
        o = (options or TransferOptions())._c()
        _check(entry(self._h, len(ranks), hs, dst, cs, len(seqs), ws, len(plan), C.byref(ls) if ls is not None else None, C.byref(o),
                     C.byref(tok)))
        return TransferCompleteNotification(self, tok.value)

    def execute_repage_batch_routed(self, sources: Mapping[int, int], dst: int, seqs: Sequence[tuple], plan: Sequence[ShardWindow],
                                    options: Optional[TransferOptions] = None, ready_flags: Optional[Mapping[int, int]] = None,
                                    layer_done_flags: int = 0, num_layers: Optional[int] = None) -> TransferCompleteNotification:
        """A decode step's new sequences, each served by its own prefill worker, as ONE hand-off
        (kvbm_manager_execute_repage_batch_routed): `execute_repage_batch` where `seqs` is a list of (tokens, {src_rank:
        src_block_ids}, dst_block_ids), the dict's keys being the source ranks the sequence is read from, under one `plan`
        (`tile_reshard_plan` over identical prefill workers, or a HeadWindow list with `num_layers`).  Each sequence is read through
        its own sources' windows only; windows of one stage may write the same destination heads as long as no sequence is routed
        to two of them.  One staged copy, one launch, one notification; with `ready_flags` (source rank -> flags) it streams as
        `execute_repage_batch` does, and only the sources some sequence names are waited on."""
        return self._repage_batch_routed(lib().kvbm_manager_execute_repage_batch_routed, sources, dst, seqs, plan, options, ready_flags,
                                         layer_done_flags, num_layers)

    def execute_repage_batch_routed_anypage(self, sources: Mapping[int, int], dst: int, seqs: Sequence[tuple], plan: Sequence[ShardWindow],
                                            options: Optional[TransferOptions] = None, ready_flags: Optional[Mapping[int, int]] = None,
                                            layer_done_flags: int = 0, num_layers: Optional[int] = None) -> TransferCompleteNotification:
        """`execute_repage_batch_routed` between engines whose page sizes need not divide each other
        (kvbm_manager_execute_repage_batch_routed_anypage), e.g. a decode step pulling each sequence from the hybrid prefill worker
        (544-token blocks) that served it into 64-token pages: the same arguments, plans, errors and streaming.  Pages past the
        exactness bound (big + small - gcd) * small < 2^32 raise UNSUPPORTED.  With dividing pages the destination bytes are
        `execute_repage_batch_routed`'s."""
        return self._repage_batch_routed(lib().kvbm_manager_execute_repage_batch_routed_anypage, sources, dst, seqs, plan, options,
                                         ready_flags, layer_done_flags, num_layers)

    def _repage_batch_routed(self, entry, sources, dst, seqs, plan, options, ready_flags, layer_done_flags, num_layers):
        """The body of `execute_repage_batch_routed` and `execute_repage_batch_routed_anypage`: `entry` is the C entry they call."""
        if plan and isinstance(plan[0], HeadWindow):
            if num_layers is None:
                raise ValueError("a HeadWindow plan needs num_layers, the destination's layer count")
            plan = [ShardWindow(w.src_rank, 0, 0, num_layers, w.src_head_begin, w.dst_head_begin, w.head_count) for w in plan]
        ranks = sorted({w.src_rank for w in plan})
        index = {r: i for i, r in enumerate(ranks)}
        hs = (C.c_uint64 * max(1, len(ranks)))(*[sources[r] for r in ranks])
        ws = self._shard_windows(ranks, plan)
        keep, cs = [], (_CRepageRouteSeq * max(1, len(seqs)))()
        for c, (tokens, src_ids, dst_ids) in zip(cs, seqs):
            if tokens.step != 1:
                raise ValueError("tokens must be a range with step 1")
            n_src = len(next(iter(src_ids.values()))) if src_ids else 0
            if any(len(x) != n_src for x in src_ids.values()):
                raise KvbmError(ErrorCode.LENGTH_MISMATCH, "the sources' block id lists have different lengths")
            if any(r not in index for r in src_ids):
                raise ValueError(f"source ranks {sorted(set(src_ids) - set(index))} are read by no window of the plan")
            arrays = {index[r]: _size_array(x)[0] for r, x in src_ids.items()}
            d, n_dst = _size_array(dst_ids)
            sp = (C.c_void_p * max(1, len(ranks)))(*[(a.addr if type(a) is _NpView else C.addressof(a)) if (a := arrays.get(i)) is not None
                                                     else None for i in range(len(ranks))])
            keep += [arrays, d, sp]
            c.token_begin, c.token_end, c.src_ids, c.n_src = tokens.start, tokens.stop, C.addressof(sp), n_src
            c.dst_ids, c.n_dst = (d.addr if type(d) is _NpView else C.addressof(d)), n_dst
            c.src_mask = sum(1 << i for i in arrays)
        ls = self._layer_stream(ranks, ready_flags, layer_done_flags) if ready_flags is not None else None
        tok = C.c_uint64()
        o = (options or TransferOptions())._c()
        _check(entry(self._h, len(ranks), hs, dst, cs, len(seqs), ws, len(plan), C.byref(ls) if ls is not None else None, C.byref(o),
                     C.byref(tok)))
        return TransferCompleteNotification(self, tok.value)

    def execute_repage_scatter(self, src: int, src_block_ids: Sequence[int], dsts: Sequence[int], dst_block_ids: Sequence[Sequence[int]],
                               plan: Sequence[ScatterWindow], tokens: range,
                               options: Optional[TransferOptions] = None) -> TransferCompleteNotification:
        """One prefill rank's KV to every decode rank that needs it, as ONE hand-off (kvbm_manager_execute_repage_scatter): heads and
        layers of `src` land in `dsts[w.dst_rank]` as each plan entry says (`tp_pp_scatter_plan` passes as it is), over `tokens`.
        `src_block_ids` is the source table's entries tokens.start // Ps .. ceil(tokens.stop / Ps), `dst_block_ids[d]` destination
        d's for its page Pd (one Pd for every destination).  Each source vector is read once and cast once, however many windows
        take it.  The options' layer range and cast scales count SOURCE layers; `options.per_dst_done_flags` is indexed like
        `dsts`; `options.done_flag` and the notification complete once, after every destination landed."""
        args = self._scatter_args(src, src_block_ids, dsts, dst_block_ids, plan, tokens)
        tok = C.c_uint64()
        o = (options or TransferOptions())._c()
        _check(lib().kvbm_manager_execute_repage_scatter(self._h, *args, C.byref(o), C.byref(tok)))
        return TransferCompleteNotification(self, tok.value)

    def execute_repage_scatter_streamed(self, src: int, src_block_ids: Sequence[int], dsts: Sequence[int],
                                        dst_block_ids: Sequence[Sequence[int]], plan: Sequence[ScatterWindow], tokens: range, ready_flags: int,
                                        options: Optional[TransferOptions] = None, layer_done_flags: int = 0) -> TransferCompleteNotification:
        """`execute_repage_scatter` streamed layer by layer (kvbm_manager_execute_repage_scatter_streamed): `ready_flags` is the
        address of the source's [num_layers] u32 ready flags, and source layer l is read only after flag l has reached
        `options.epoch`, so the push overlaps the prefill's forward pass; `layer_done_flags` (an address, or 0) gets entry l =
        epoch once source layer l landed in every destination.  Options: those of `execute_repage_scatter`, plus epoch, gate_mode,
        gate_timeout_ms and max_ctas; `per_dst_done_flags` and `done_flag` are written after the last byte, never after a gate
        timeout.  The bytes and bytes_moved are `execute_repage_scatter`'s."""
        args = self._scatter_args(src, src_block_ids, dsts, dst_block_ids, plan, tokens)
        ls = self._layer_stream([0], {0: ready_flags}, layer_done_flags)
        tok = C.c_uint64()
        o = (options or TransferOptions())._c()
        _check(lib().kvbm_manager_execute_repage_scatter_streamed(self._h, *args, C.byref(ls), C.byref(o), C.byref(tok)))
        return TransferCompleteNotification(self, tok.value)

    def execute_repage_scatter_batch(self, src: int, dsts: Sequence[int], seqs: Sequence[tuple], plan: Sequence[ScatterWindow],
                                     options: Optional[TransferOptions] = None, ready_flags: Optional[int] = None,
                                     layer_done_flags: int = 0) -> TransferCompleteNotification:
        """A prefill batch's sequences pushed to every decode rank that needs them, as ONE hand-off
        (kvbm_manager_execute_repage_scatter_batch): `seqs` is a list of (tokens, src_block_ids, [dst_block_ids per destination]),
        each what `execute_repage_scatter` takes for one request, under one `plan` (`tp_pp_scatter_plan` passes as it is).  One
        staged copy of every table, one launch, one notification; `options.per_dst_done_flags` and `options.done_flag` are written
        once, after every sequence landed.  With `ready_flags` (the address of the source's [num_layers] u32 ready flags) it streams
        as `execute_repage_scatter_streamed` does, and `layer_done_flags[l]` is written once source layer l of every sequence
        landed.  Two sequences may share source blocks; a destination block may appear once per destination in the whole batch.
        The first rejected sequence raises what `execute_repage_scatter` would raise for it."""
        return self._repage_scatter_batch(lib().kvbm_manager_execute_repage_scatter_batch, src, dsts, seqs, plan, options, ready_flags,
                                          layer_done_flags)

    def execute_repage_scatter_anypage(self, src: int, dsts: Sequence[int], seqs: Sequence[tuple], plan: Sequence[ScatterWindow],
                                       options: Optional[TransferOptions] = None, ready_flags: Optional[int] = None,
                                       layer_done_flags: int = 0) -> TransferCompleteNotification:
        """`execute_repage_scatter_batch` between engines whose page sizes need not divide each other
        (kvbm_manager_execute_repage_scatter_anypage), e.g. a hybrid model's 544-token attention block pushed into 64-token decode
        pages, or 24 into 16: the same arguments, plans, errors and streaming.  Pages past the exactness bound
        (big + small - gcd) * small < 2^32 raise UNSUPPORTED.  With dividing pages the destination bytes are
        `execute_repage_scatter_batch`'s."""
        return self._repage_scatter_batch(lib().kvbm_manager_execute_repage_scatter_anypage, src, dsts, seqs, plan, options, ready_flags,
                                          layer_done_flags)

    def _repage_scatter_batch(self, entry, src, dsts, seqs, plan, options, ready_flags, layer_done_flags):
        """The body of `execute_repage_scatter_batch` and `execute_repage_scatter_anypage`: `entry` is the C entry they call."""
        keep, cs, ws = [], (_CScatterBatchSeq * max(1, len(seqs)))(), None
        for c, (tokens, src_ids, dst_ids) in zip(cs, seqs):
            args = self._scatter_args(src, src_ids, dsts, dst_ids, plan, tokens)
            _, s, ns, _, _, dp, n_dst, tb, te, ws, _ = args
            keep.append(args)
            c.token_begin, c.token_end, c.src_ids, c.n_src = tb, te, s if isinstance(s, int) else C.addressof(s), ns
            c.dst_ids, c.n_dst = C.addressof(dp), n_dst
        if ws is None:
            ws = self._scatter_args(src, [], dsts, [[]] * len(dsts), plan, range(0, 0))[9]
        hs = (C.c_uint64 * max(1, len(dsts)))(*dsts)
        ls = self._layer_stream([0], {0: ready_flags}, layer_done_flags) if ready_flags is not None else None
        tok = C.c_uint64()
        o = (options or TransferOptions())._c()
        _check(entry(self._h, src, len(dsts), hs, cs, len(seqs), ws, len(plan), C.byref(ls) if ls is not None else None, C.byref(o),
                     C.byref(tok)))
        return TransferCompleteNotification(self, tok.value)

    def execute_repage_scatter_routed(self, src: int, dsts: Sequence[int], seqs: Sequence[tuple], plan: Sequence[ScatterWindow],
                                      options: Optional[TransferOptions] = None, ready_flags: Optional[int] = None,
                                      layer_done_flags: int = 0) -> TransferCompleteNotification:
        """A prefill batch whose sequences go to different decode workers, as ONE hand-off (kvbm_manager_execute_repage_scatter_routed):
        `seqs` is a list of (tokens, src_block_ids, {dst_index: dst_block_ids}), the dict's keys being the destinations (indices
        into `dsts`) the sequence goes to, under one `plan` (`tile_scatter_plan` over identical workers).  Each sequence lands in
        its own destinations only; every other destination byte keeps its value.  One staged copy, one launch, one notification;
        `options.per_dst_done_flags` and `options.done_flag` are written once, after every sequence landed.  With `ready_flags` it
        streams as `execute_repage_scatter_batch` does.  A destination block may appear once per destination among the sequences
        routed to it."""
        return self._repage_scatter_routed(lib().kvbm_manager_execute_repage_scatter_routed, src, dsts, seqs, plan, options, ready_flags,
                                           layer_done_flags)

    def execute_repage_scatter_routed_anypage(self, src: int, dsts: Sequence[int], seqs: Sequence[tuple], plan: Sequence[ScatterWindow],
                                              options: Optional[TransferOptions] = None, ready_flags: Optional[int] = None,
                                              layer_done_flags: int = 0) -> TransferCompleteNotification:
        """`execute_repage_scatter_routed` between engines whose page sizes need not divide each other
        (kvbm_manager_execute_repage_scatter_routed_anypage), e.g. a hybrid prefill pool's 544-token blocks pushed to several decode
        workers with 64-token pages, each sequence to its own worker: the same arguments, plans, errors and streaming.  Pages past
        the exactness bound (big + small - gcd) * small < 2^32 raise UNSUPPORTED.  With dividing pages the destination bytes are
        `execute_repage_scatter_routed`'s."""
        return self._repage_scatter_routed(lib().kvbm_manager_execute_repage_scatter_routed_anypage, src, dsts, seqs, plan, options,
                                           ready_flags, layer_done_flags)

    def _repage_scatter_routed(self, entry, src, dsts, seqs, plan, options, ready_flags, layer_done_flags):
        """The body of `execute_repage_scatter_routed` and `execute_repage_scatter_routed_anypage`: `entry` is the C entry they
        call."""
        keep, cs = [], (_CScatterRouteSeq * max(1, len(seqs)))()
        for c, (tokens, src_ids, routed) in zip(cs, seqs):
            if tokens.step != 1:
                raise ValueError("tokens must be a range with step 1")
            n_dst = len(next(iter(routed.values()))) if routed else 0
            if any(len(x) != n_dst for x in routed.values()):
                raise KvbmError(ErrorCode.LENGTH_MISMATCH, "the destinations' block id lists have different lengths")
            s, ns = _size_array(src_ids)
            arrays = {d: _size_array(x)[0] for d, x in routed.items() if 0 <= d < len(dsts)}
            PP = C.POINTER(C.c_size_t)
            as_ptr = lambda a: a._as_parameter_ if isinstance(a, _NpView) else C.cast(a, PP)  # noqa: E731
            dp = (PP * max(1, len(dsts)))(*[as_ptr(arrays[d]) if d in arrays else None for d in range(len(dsts))])
            keep.append((s, arrays, dp))
            if any(not 0 <= d < 32 for d in routed):
                raise ValueError(f"destination indices {sorted(routed)} do not fit a 32-bit mask")
            c.token_begin, c.token_end, c.n_src, c.n_dst = tokens.start, tokens.stop, ns, n_dst
            c.dst_mask = sum(1 << d for d in routed)
            c.src_ids = s.addr if type(s) is _NpView else C.addressof(s)
            c.dst_ids = C.addressof(dp)
        ws = (_CScatterWindow * max(1, len(plan)))(*[_CScatterWindow(w.dst_rank, w.src_layer_begin, w.dst_layer_begin, w.layer_count,
                                                                     w.src_head_begin, w.dst_head_begin, w.head_count) for w in plan])
        hs = (C.c_uint64 * max(1, len(dsts)))(*dsts)
        ls = self._layer_stream([0], {0: ready_flags}, layer_done_flags) if ready_flags is not None else None
        tok = C.c_uint64()
        o = (options or TransferOptions())._c()
        _check(entry(self._h, src, len(dsts), hs, cs, len(seqs), ws, len(plan), C.byref(ls) if ls is not None else None, C.byref(o),
                     C.byref(tok)))
        return TransferCompleteNotification(self, tok.value)

    @staticmethod
    def _scatter_args(src: int, src_block_ids: Sequence[int], dsts: Sequence[int], dst_block_ids: Sequence[Sequence[int]],
                      plan: Sequence[ScatterWindow], tokens: range) -> tuple:
        """The C arguments of a scatter from `src` through the window count; the arrays they point to stay alive with the tuple."""
        if tokens.step != 1:
            raise ValueError("tokens must be a range with step 1")
        if len(dst_block_ids) != len(dsts):
            raise ValueError(f"{len(dst_block_ids)} destination id lists for {len(dsts)} destinations")
        s, ns = _size_array(src_block_ids)
        n_dst = len(dst_block_ids[0]) if dsts else 0
        if any(len(x) != n_dst for x in dst_block_ids):
            raise KvbmError(ErrorCode.LENGTH_MISMATCH, "the destinations' block id lists have different lengths")
        hs = (C.c_uint64 * max(1, len(dsts)))(*dsts)
        d_arrays = [_size_array(x)[0] for x in dst_block_ids]
        PP = C.POINTER(C.c_size_t)
        as_ptr = lambda a: a._as_parameter_ if isinstance(a, _NpView) else C.cast(a, PP)  # noqa: E731
        dp = (PP * max(1, len(dsts)))(*[as_ptr(a) for a in d_arrays])
        dp._keep = d_arrays
        ws = (_CScatterWindow * max(1, len(plan)))(*[_CScatterWindow(w.dst_rank, w.src_layer_begin, w.dst_layer_begin, w.layer_count,
                                                                     w.src_head_begin, w.dst_head_begin, w.head_count) for w in plan])
        return (src, s.addr if type(s) is _NpView else s, ns, len(dsts), hs, dp, n_dst, tokens.start, tokens.stop, ws, len(plan))

    def execute_fanout(self, src: int, dsts: Sequence[int], src_block_ids: Sequence[Sequence[int]],
                       dst_block_ids: Sequence[Sequence[int]], replicate: bool = False,
                       options: Optional[TransferOptions] = None) -> TransferCompleteNotification:
        nd = len(dsts)
        n = len(dst_block_ids[0])
        if any(len(x) != n for x in dst_block_ids) or any(len(x) != n for x in src_block_ids):
            raise KvbmError(ErrorCode.LENGTH_MISMATCH, "Block ID lists have mismatched lengths")
        hs = (C.c_uint64 * nd)(*dsts)
        s_arrays = [_size_array(x)[0] for x in (src_block_ids if not replicate else [src_block_ids[0]] * nd)]
        d_arrays = [_size_array(x)[0] for x in dst_block_ids]
        PP = C.POINTER(C.c_size_t)
        as_ptr = lambda a: a._as_parameter_ if isinstance(a, _NpView) else C.cast(a, PP)  # noqa: E731
        sp = (PP * nd)(*[as_ptr(a) for a in s_arrays])
        dp = (PP * nd)(*[as_ptr(a) for a in d_arrays])
        tok = C.c_uint64()
        o = (options or TransferOptions())._c()
        _check(lib().kvbm_manager_execute_fanout(self._h, src, nd, hs, sp, dp, n, int(replicate), C.byref(o), C.byref(tok)))
        return TransferCompleteNotification(self, tok.value)

    def broadcast(self, src: int, dsts: Sequence[int], src_block_ids: Sequence[int],
                  dst_block_ids: Sequence[int], layer_range: Optional[range] = None) -> TransferCompleteNotification:
        """CollectiveOps::broadcast (lib/kvbm-engine/src/collectives/mod.rs:99-106): same blocks, same destination
        ids on every rank -- here one replicate launch over peer mappings instead of grouped ncclBcast."""
        return self.execute_fanout(src, dsts, [src_block_ids] * len(dsts), [dst_block_ids] * len(dsts), replicate=True,
                                   options=TransferOptions(layer_range=layer_range))

    def set_capabilities(self, allow_gds: bool = False, allow_gpu_rdma: bool = True) -> None:
        """TransferCapabilities (strategy.rs:245-278); allow_gpu_rdma=False turns cross-GPU transfers into the reference's
        TwoHop plan through `TransferOptions.bounce_buffer`."""
        caps = _CCaps(int(allow_gds), int(allow_gpu_rdma))
        _check(lib().kvbm_manager_set_capabilities(self._h, C.byref(caps)))

    def bytes_moved(self) -> int:
        return lib().kvbm_manager_bytes_moved(self._h)

    def h2d_bytes(self) -> int:
        return lib().kvbm_manager_h2d_bytes(self._h)


def multicast_supported(device: int = 0) -> bool:
    """CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED (NVSwitch multicast objects usable from this process)."""
    return bool(lib().kvbm_mc_supported(device))


class MulticastGroup:
    """NVLS multicast group (`kvbm_mc_group_*`, include/kvbm_physical.h): the receivers' pools are bound to one
    multicast object; the sender maps it and transfers with `TransferOptions(multicast=1)`, so identical KV blocks reach
    every bound GPU with ONE write per tile -- the replacement of the grouped `ncclBcast` per region
    (lib/kvbm-engine/src/collectives/nccl.rs:421-462).

    Call order across all participants: create()/from_fd() -> add_device() for every device (by its owning process)
    -> barrier -> bind_local() on every receiver -> barrier -> map() on the sender."""

    def __init__(self, handle: int, num_devices: int):
        self._h = C.c_void_p(handle)
        self.num_devices = num_devices

    @staticmethod
    def create(num_devices: int, bytes_per_device: int, shareable: bool = False) -> "MulticastGroup":
        h = C.c_void_p()
        _check(lib().kvbm_mc_group_create(num_devices, bytes_per_device, int(shareable), C.byref(h)))
        return MulticastGroup(h.value, num_devices)

    @staticmethod
    def from_fd(fd: int, num_devices: int, bytes_per_device: int) -> "MulticastGroup":
        h = C.c_void_p()
        _check(lib().kvbm_mc_group_import_fd(fd, num_devices, bytes_per_device, C.byref(h)))
        return MulticastGroup(h.value, num_devices)

    @property
    def size(self) -> int:
        return lib().kvbm_mc_group_size(self._h)

    def export_fd(self) -> int:
        fd = C.c_int(-1)
        _check(lib().kvbm_mc_group_export_fd(self._h, C.byref(fd)))
        return fd.value

    def add_device(self, device: int) -> None:
        _check(lib().kvbm_mc_group_add_device(self._h, device))

    def bind_local(self, device: int) -> int:
        """Allocate + bind this device's pool; returns its ordinary (unicast) device address."""
        p = C.c_void_p()
        _check(lib().kvbm_mc_group_bind_local(self._h, device, C.byref(p)))
        return p.value

    def bind_addr(self, device: int, ptr: int, nbytes: int) -> None:
        """Bind memory the engine already owns (cuMemCreate-backed, granularity-aligned) instead of a pool allocated here."""
        _check(lib().kvbm_mc_group_bind_addr(self._h, device, ptr, nbytes))

    def map(self, device: int) -> int:
        """Map the multicast object for the sending device; returns the multicast address of offset 0."""
        p = C.c_void_p()
        _check(lib().kvbm_mc_group_map(self._h, device, C.byref(p)))
        return p.value

    def close(self) -> None:
        if self._h:
            lib().kvbm_mc_group_destroy(self._h)
            self._h = C.c_void_p()

    def detach(self) -> None:
        """Forget the group without tearing it down (the driver reclaims it at process exit).  Unbinding a multicast
        object takes the driver seconds; a process that is about to exit need not wait for it."""
        self._h = C.c_void_p()

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass
