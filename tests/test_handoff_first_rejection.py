"""The first rejection of a manager hand-off that fails several checks at once, on a host-only manager.  Each entry's own host
tests fault one check at a time; these requests fail two or more, so they pin the order in which every entry makes its checks:
each case names the code and a fragment of the text the first failing check reports."""
import ctypes as C

import numpy as np
import pytest

from dynamo_b200 import kernels as K
from dynamo_b200 import physical as P
from dynamo_b200.physical import ErrorCode, HeadWindow, KvbmError, ShardWindow, StorageKind, TransferOptions
from tests.test_repage_host import host_mgr  # noqa: F401  (the host-only manager fixture)

KV = K.KvBlockLayout
BAD = 0xDEAD
PP = C.POINTER(C.c_size_t)
NUL = (PP * 1)(None)   # one source, no id list


def _first(fn, code, fragment):
    with pytest.raises(KvbmError) as e:
        fn()
    assert (e.value.code, fragment in e.value.msg) == (code, True), (e.value.code, e.value.msg)


def _c_first(rc, code, fragment):
    msg = P.lib().kvbm_last_error().decode()
    assert (rc, fragment in msg) == (code, True), (rc, msg)


def _ids(*v):
    return (C.c_size_t * len(v))(*v)


def _handles(*h):
    return (C.c_uint64 * len(h))(*h)


def _windows(*w):
    return (P._CHeadWindow * len(w))(*[P._CHeadWindow(*x) for x in w])


def _pageable_flags():
    return np.zeros(8, np.uint32)


# ---------------------------------------------------------------------------------------------------------------------
# execute_transfer / execute_fanout
# ---------------------------------------------------------------------------------------------------------------------
def test_transfer_first_rejection(host_mgr):  # noqa: F811
    mgr, reg = host_mgr
    s, d = reg(16), reg(16)
    go = lambda src, dst, o=None: lambda: mgr.execute_transfer(src, [0], dst, [1], o)  # noqa: E731
    _first(go(BAD, BAD), ErrorCode.HANDLE, "invalid source handle")
    # a head window past the source's heads and a layer range past its layers: the window is the pair's check
    _first(go(s, d, TransferOptions(head_window=(3, 0, 2), layer_range=range(0, 3))), ErrorCode.RANGE, "Head window")
    # a layer range past the pools' layers and scales without a cast
    _first(go(s, d, TransferOptions(layer_range=range(0, 3), cast_scales=np.ones(4, np.float32))), ErrorCode.RANGE, "Layer range")
    # an unnamed source format under a head window and a layer range past the layers
    u = reg(16, kv=None)
    _first(go(u, d, TransferOptions(head_window=(0, 0, 2), layer_range=range(0, 3))), ErrorCode.UNSUPPORTED,
           "Layout transformation not supported")


def test_fanout_first_rejection(host_mgr):  # noqa: F811
    mgr, reg = host_mgr
    s, d0, d1 = reg(16), reg(16), reg(16)
    go = lambda dsts, o=None: lambda: mgr.execute_fanout(s, dsts, [[0]] * len(dsts), [[1]] * len(dsts), False, o)  # noqa: E731
    _first(go([d0] * 9), ErrorCode.ERR, "number of destinations")
    # destination 0 with other layer counts, destination 1 an invalid handle: destination 0's pair first
    _first(go([reg(16, nl=3), BAD]), ErrorCode.INCOMPATIBLE, "layer counts")
    # destination 1 an invalid handle, a layer range past the layers
    _first(go([d0, BAD], TransferOptions(layer_range=range(0, 3))), ErrorCode.HANDLE, "invalid destination handle")
    # a layout transformation with two destinations, and a layer range past the layers
    _first(go([d0, d1], TransferOptions(dst_kv_layout=int(KV.UniversalTP), layer_range=range(0, 3))), ErrorCode.UNSUPPORTED,
           "one destination")


# ---------------------------------------------------------------------------------------------------------------------
# execute_gather / execute_gather_streamed
# ---------------------------------------------------------------------------------------------------------------------
def test_gather_first_rejection(host_mgr):  # noqa: F811
    mgr, reg = host_mgr
    s0, s1, d = reg(16, nh=2), reg(16, nh=2), reg(16, nh=4)
    src = {0: (s0, [0]), 1: (s1, [1])}
    go = lambda plan, dst=d, sources=src, o=None: lambda: mgr.execute_gather(sources, dst, [2], plan, o)  # noqa: E731
    # windows that overlap in the destination, and an invalid destination handle
    _first(go([HeadWindow(0, 0, 0, 2), HeadWindow(1, 0, 1, 2)], dst=BAD), ErrorCode.OVERLAP, "overlap in the destination")
    # null id lists and an invalid destination handle
    rc = P.lib().kvbm_manager_execute_gather(mgr._h, 1, _handles(s0), None, BAD, None, 1, _windows((0, 0, 0, 2)), 1,
                                             C.byref(P._COptions()), None)
    _c_first(rc, ErrorCode.ERR, "null block id list")
    # both handles invalid, and a window past the source's heads
    _first(go([HeadWindow(0, 1, 0, 2)], dst=BAD, sources={0: (BAD, [0])}), ErrorCode.HANDLE, "invalid source handle")
    # an invalid destination handle, and a window past the source's heads
    _first(go([HeadWindow(0, 1, 0, 2)], dst=BAD), ErrorCode.HANDLE, "invalid destination handle")
    # a window past the source's heads, and a layer range past the layers
    _first(go([HeadWindow(0, 1, 0, 2)], o=TransferOptions(layer_range=range(0, 3))), ErrorCode.RANGE, "Head window")
    # source 1's pair fails a check, source 0's window has a layer range past its layers: source 0 first
    _first(go([HeadWindow(0, 0, 0, 2), HeadWindow(1, 0, 2, 2)], sources={0: (s0, [0]), 1: (reg(16, nh=2, nl=3), [1])},
              o=TransferOptions(layer_range=range(0, 3))), ErrorCode.RANGE, "Layer range")


def test_gather_streamed_first_rejection(host_mgr):  # noqa: F811
    mgr, reg = host_mgr
    s0, s1, d = reg(16, nh=2), reg(16, nh=2), reg(16, nh=4)
    src = {0: (s0, [0]), 1: (s1, [1])}
    plan = [HeadWindow(0, 0, 0, 2), HeadWindow(1, 0, 2, 2)]
    flags = _pageable_flags()
    go = lambda p, ready, dst=d: lambda: mgr.execute_gather_streamed(src, dst, [2], p, ready)  # noqa: E731
    # a source without ready flags, and an invalid destination handle
    _first(go(plan, {0: flags.ctypes.data}, dst=BAD), ErrorCode.ERR, "no layer ready flags")
    # a source without ready flags, and windows that overlap in the destination
    _first(go([plan[0], HeadWindow(1, 0, 1, 2)], {0: flags.ctypes.data}), ErrorCode.ERR, "no layer ready flags")
    # pageable flags the device cannot read, on a manager without a device: the missing device first
    _first(go(plan, {0: flags.ctypes.data, 1: flags.ctypes.data}), ErrorCode.CUDA, "without a CUDA device")
    # a stream naming one source for a request with two, and an invalid destination handle
    fl = (C.c_void_p * 1)(flags.ctypes.data)
    ls = P._CLayerStream(C.cast(fl, C.c_void_p), 1, None)
    rc = P.lib().kvbm_manager_execute_gather_streamed(mgr._h, 2, _handles(s0, s1), None, BAD, None, 0,
                                                      _windows((0, 0, 0, 2), (1, 0, 2, 2)), 2, C.byref(ls), C.byref(P._COptions()), None)
    _c_first(rc, ErrorCode.LENGTH_MISMATCH, "names 1 sources' ready flags")


# ---------------------------------------------------------------------------------------------------------------------
# execute_stage_gather, with and without a layer stream
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def stage(host_mgr):  # noqa: F811
    """Stage 0: layers 0..3 of a and b (heads 0-1 and 2-3); stage 1: layers 0..5 of c as destination layers 3..8."""
    mgr, reg = host_mgr
    a, b, c, d = reg(16, nh=2, nl=3), reg(16, nh=2, nl=3), reg(16, nh=2, nl=5), reg(16, nh=4, nl=8)
    plan = [ShardWindow(0, 0, 0, 3, 0, 0, 2), ShardWindow(1, 0, 0, 3, 0, 2, 2), ShardWindow(2, 0, 3, 5, 0, 0, 2),
            ShardWindow(2, 0, 3, 5, 0, 2, 2)]
    return mgr, reg, {0: (a, [0]), 1: (b, [1]), 2: (c, [2])}, d, plan


def test_stage_gather_first_rejection(stage):
    mgr, reg, src, d, plan = stage
    go = lambda p, dst=d, o=None: lambda: mgr.execute_stage_gather(src, dst, [3], p, o)  # noqa: E731
    # null id lists and an invalid destination handle
    sw = (P._CShardWindow * 1)(P._CShardWindow(0, 0, 0, 3, 0, 0, 2))
    rc = P.lib().kvbm_manager_execute_stage_gather(mgr._h, 1, _handles(src[0][0]), None, BAD, None, 1, sw, 1, None,
                                                   C.byref(P._COptions()), None)
    _c_first(rc, ErrorCode.ERR, "null block id list")
    # an invalid destination handle, and a window past its source's layers
    _first(go([ShardWindow(0, 1, 0, 3, 0, 0, 2)] + plan[1:], dst=BAD), ErrorCode.HANDLE, "invalid destination handle")
    # windows past the destination's layers, and a head window past their source's heads
    _first(go(plan[:2] + [ShardWindow(2, 0, 4, 5, 1, 0, 2), ShardWindow(2, 0, 4, 5, 1, 2, 2)]), ErrorCode.RANGE,
           "destination's num_layers")
    # destination layers 3..8 in no window, and a layer range past the destination's layers
    _first(go(plan[:2], o=TransferOptions(layer_range=range(0, 9))), ErrorCode.RANGE, "destination layer 3")
    # a head window past a source's heads, and a layer range past the destination's layers
    _first(go([ShardWindow(0, 0, 0, 3, 1, 0, 2)] + plan[1:], o=TransferOptions(layer_range=range(0, 9))), ErrorCode.RANGE,
           "Head window")
    # a layer range past the destination's layers, and scales without a cast
    _first(go(plan, o=TransferOptions(layer_range=range(0, 9), cast_scales=np.ones(4, np.float32))), ErrorCode.RANGE,
           "exceeds num_layers 8")
    # scales without a cast, and too few of them for the destination's layers
    _first(go(plan, o=TransferOptions(cast_scales=np.ones(4, np.float32))), ErrorCode.ERR, "need a cast_mode")


def test_stage_gather_streamed_first_rejection(stage):
    mgr, reg, src, d, plan = stage
    flags = _pageable_flags()
    f = flags.ctypes.data
    go = lambda p, ready, dst=d: lambda: mgr.execute_stage_gather(src, dst, [3], p, None, ready_flags=ready)  # noqa: E731
    # a source without ready flags, and an invalid destination handle
    _first(go(plan, {0: f, 1: f}, dst=BAD), ErrorCode.ERR, "no layer ready flags")
    # a source without ready flags, and a window past its source's layers
    _first(go([ShardWindow(0, 1, 0, 3, 0, 0, 2)] + plan[1:], {0: f, 2: f}), ErrorCode.ERR, "no layer ready flags")
    # pageable flags the device cannot read, on a manager without a device: the missing device first
    _first(go(plan, {0: f, 1: f, 2: f}), ErrorCode.CUDA, "without a CUDA device")
    # flags on host pools, whose strategy is Memcpy: the strategy first
    h = [reg(16, nh=2, nl=3, storage=StorageKind.System) for _ in range(2)] + [reg(16, nh=2, nl=5, storage=StorageKind.System)]
    hd = reg(16, nh=4, nl=8, storage=StorageKind.System)
    e = lambda: mgr.execute_stage_gather({r: (h[r], src[r][1]) for r in range(3)}, hd, [3], plan, None,  # noqa: E731
                                         ready_flags={0: f, 1: f, 2: f})
    _first(e, ErrorCode.UNSUPPORTED, "CUDA strategies")


# ---------------------------------------------------------------------------------------------------------------------
# execute_repage
# ---------------------------------------------------------------------------------------------------------------------
def test_repage_first_rejection(host_mgr):  # noqa: F811
    mgr, reg = host_mgr
    s, d = reg(16, nh=2), reg(64, nh=2)
    go = lambda src=s, dst=d, sid=(0, 1, 2), did=(3,), tok=range(5, 40), o=None: (  # noqa: E731
        lambda: mgr.execute_repage(src, list(sid), dst, list(did), tok, o))
    _first(go(src=BAD, dst=BAD), ErrorCode.HANDLE, "invalid source handle")
    # an invalid destination handle, and a source in an unnamed format
    _first(go(src=reg(16, nh=2, kv=None), dst=BAD), ErrorCode.HANDLE, "invalid destination handle")
    # a head window in the options, and pages that do not divide
    _first(go(dst=reg(24, nh=2), did=(0,), o=TransferOptions(head_window=(0, 0, 2))), ErrorCode.UNSUPPORTED,
           "re-paging transfer takes no")
    # other head counts, and a layer range past the layers
    _first(go(dst=reg(64, nh=4), o=TransferOptions(layer_range=range(0, 3))), ErrorCode.INCOMPATIBLE, "equal num_heads")
    # a layer range past the layers, and ids that do not match the token range
    _first(go(sid=(0, 1), o=TransferOptions(layer_range=range(0, 3))), ErrorCode.RANGE, "Layer range")
    # ids that do not match the token range, and ids past the destination's blocks
    _first(go(sid=(0, 1), did=(9,)), ErrorCode.LENGTH_MISMATCH, "3 source and 1 destination")
    # a null source id list, and a destination id past its blocks
    rc = P.lib().kvbm_manager_execute_repage(mgr._h, s, None, 3, d, _ids(9), 1, 5, 40, C.byref(P._COptions()), None)
    _c_first(rc, ErrorCode.ERR, "null block id list")
    # host pools, whose strategy is Memcpy, on a manager without a device: the strategy first
    hs, hd = reg(16, nh=2, storage=StorageKind.System), reg(64, nh=2, storage=StorageKind.System)
    _first(go(src=hs, dst=hd), ErrorCode.UNSUPPORTED, "direct CUDA strategy")


# ---------------------------------------------------------------------------------------------------------------------
# execute_repage_gather / execute_repage_gather_streamed
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def repage_gather(host_mgr):  # noqa: F811
    """TP2 at page 16 (2 heads per rank) -> TP1 at page 64 (4 heads); tokens 5..40: 3 source blocks, 1 destination block."""
    mgr, reg = host_mgr
    s0, s1, d = reg(16, nh=2), reg(16, nh=2), reg(64, nh=4)
    plan = [HeadWindow(0, 0, 0, 2), HeadWindow(1, 0, 2, 2)]
    return mgr, reg, {0: (s0, [0, 1, 2]), 1: (s1, [3, 4, 5])}, d, plan


def test_repage_gather_first_rejection(repage_gather):
    mgr, reg, src, d, plan = repage_gather
    go = lambda p=plan, sources=src, dst=d, o=None: lambda: mgr.execute_repage_gather(sources, dst, [3], p, range(5, 40), o)  # noqa: E731
    # a window without heads, and an invalid destination handle
    _first(go(p=[HeadWindow(0, 0, 0, 0), plan[1]], dst=BAD), ErrorCode.RANGE, "has no heads")
    # a head window in the options, and an invalid destination handle: the gather's text
    _first(go(dst=BAD, o=TransferOptions(head_window=(0, 0, 2))), ErrorCode.ERR, "options.head_count must be 0")
    # both handles invalid: the destination first
    _first(go(sources={0: (BAD, [0, 1, 2]), 1: (src[1][0], [3, 4, 5])}, dst=BAD), ErrorCode.HANDLE, "invalid destination handle")
    # source 0 in an unnamed format, source 1 an invalid handle
    _first(go(sources={0: (reg(16, nh=2, kv=None), [0, 1, 2]), 1: (BAD, [3, 4, 5])}), ErrorCode.UNSUPPORTED, "named KV block layouts")
    # source 0's window past its heads, source 1 with another page size
    _first(go(p=[HeadWindow(0, 1, 0, 2), plan[1]], sources={0: src[0], 1: (reg(32, nh=2), [3, 4, 5])}), ErrorCode.RANGE, "Head window")
    # a layer range past the layers, and ids that do not match the token range
    _first(go(sources={0: (src[0][0], [0, 1]), 1: (src[1][0], [3, 4])}, o=TransferOptions(layer_range=range(0, 3))),
           ErrorCode.RANGE, "Layer range")
    # a null source id list, and a destination id past its blocks
    PP2 = (PP * 2)(None, None)
    rc = P.lib().kvbm_manager_execute_repage_gather(mgr._h, 2, _handles(src[0][0], src[1][0]), PP2, 3, d, _ids(9), 1, 5, 40,
                                                    _windows((0, 0, 0, 2), (1, 0, 2, 2)), 2, C.byref(P._COptions()), None)
    _c_first(rc, ErrorCode.ERR, "null block id list")
    # host pools, whose strategy is Memcpy, on a manager without a device: the strategy first
    h0, h1, hd = (reg(p, nh=n, storage=StorageKind.System) for p, n in ((16, 2), (16, 2), (64, 4)))
    _first(go(sources={0: (h0, [0, 1, 2]), 1: (h1, [3, 4, 5])}, dst=hd), ErrorCode.UNSUPPORTED, "direct CUDA strategy")


def test_repage_gather_streamed_first_rejection(repage_gather):
    mgr, reg, src, d, plan = repage_gather
    flags = _pageable_flags()
    f = flags.ctypes.data
    go = lambda p, ready, dst=d, o=None: lambda: mgr.execute_repage_gather_streamed(src, dst, [3], p, range(5, 40), ready, o)  # noqa: E731
    # a source without ready flags, and a window without heads
    _first(go([HeadWindow(0, 0, 0, 0), plan[1]], {0: f}), ErrorCode.ERR, "no layer ready flags")
    # a source without ready flags, and an invalid destination handle
    _first(go(plan, {1: f}, dst=BAD), ErrorCode.ERR, "no layer ready flags")
    # pageable flags the device cannot read, on a manager without a device: the missing device first
    _first(go(plan, {0: f, 1: f}), ErrorCode.CUDA, "without a CUDA device")
    # flags in the options, and an invalid destination handle: the gather's window checks, then the handle
    _first(go(plan, {0: f, 1: f}, dst=BAD, o=TransferOptions(layer_ready_flags=f)), ErrorCode.HANDLE, "invalid destination handle")
