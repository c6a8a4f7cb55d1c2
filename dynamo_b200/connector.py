"""Worker side of Dynamo's KVBM connector, over the H100 transfer path (SURVEY.md §8 f1).

Mirrors the surface the vLLM / TRT-LLM model runner calls through pyo3
(`PyKvConnectorWorker`, /root/reference/lib/bindings/kvbm/src/block_manager/vllm/connector/worker.rs:474-560;
trait `Worker` :27-54) and its bookkeeping (`WorkerSchedulerClient`,
lib/llm/src/block_manager/connector/scheduler.rs:83-268), with the wire formats of
`ConnectorMetadata` (lib/bindings/kvbm/src/block_manager/vllm/connector.rs:158-185),
`WorkerTransferRequest` / `LeaderTransferRequest` / `SchedulerRequirement`
(lib/llm/src/block_manager/connector/protocol.rs:60-140) and `BlockTransferRequest`
(lib/llm/src/block_manager/distributed/utils.rs:47-84) exactly as serde_json writes them.

What changes underneath:
  * bytes move through `TransferManager.execute_transfer` (one block-table kernel launch) instead of
    `BlockTransferHandler` -> per-chunk `cudaMemcpyAsync` / K1 (distributed/transfer.rs:304-395);
  * `save_kv_layer` never blocks the host: the reference waits on the last layer's event with
    `cuEventSynchronize` (worker.rs:341); here every layer's event is turned into a device-side ready flag
    by a helper stream (`cuStreamWaitEvent` + `cuStreamWriteValue32`), which is what lets ONE gated transfer
    launch stream all layers behind the forward pass;
  * completion is read from the transfer's completion word, not polled through cudaEventQuery.
The leader / ZMQ / slot manager on the scheduler side stay Dynamo's; `handle_block_transfer` is the entry point
its `BlockTransferRequest`s arrive through.
"""
from __future__ import annotations

import json
import uuid as _uuid
from dataclasses import dataclass, field
from typing import Dict, Iterable, List, Optional, Sequence, Set, Tuple

from . import kernels as K
from .physical import (BlockDimension, KvbmError, LayoutConfig, StorageKind, TransferCompleteNotification,
                       TransferManager, TransferOptions)

def stable_worker_id(worker_id) -> int:
    """Deterministic 48-bit id for a worker name (the reference's worker_id is a u64 the caller supplies,
    lib/kvbm-physical/src/manager/handle.rs:16-50).  Integers (or decimal strings) are used as they are; anything else
    is digested with BLAKE2b -- never Python's per-process randomised hash()."""
    if isinstance(worker_id, int):
        return worker_id & 0xFFFFFFFFFFFF
    text = str(worker_id)
    if text.isdigit():
        return int(text) & 0xFFFFFFFFFFFF
    import hashlib
    return int.from_bytes(hashlib.blake2b(text.encode(), digest_size=6).digest(), "little")


LOAD, STORE = "Load", "Store"
SCHEDULED, IMMEDIATE = "Scheduled", "Immediate"
DEVICE, HOST, DISK = "Device", "Host", "Disk"


# ----------------------------------------------------------------------------------------------- wire formats
@dataclass
class WorkerTransferRequest:
    """protocol.rs: `WorkerTransferRequest {request_id, uuid, transfer_type, request_type}`."""
    request_id: str
    uuid: str
    transfer_type: str   # "Load" | "Store"
    request_type: str    # "Scheduled" | "Immediate"

    def to_json(self) -> dict:
        return {"request_id": self.request_id, "uuid": self.uuid, "transfer_type": self.transfer_type,
                "request_type": self.request_type}

    @staticmethod
    def from_json(d: dict) -> "WorkerTransferRequest":
        if d["transfer_type"] not in (LOAD, STORE) or d["request_type"] not in (SCHEDULED, IMMEDIATE):
            raise ValueError(f"unknown variant in {d}")
        return WorkerTransferRequest(d["request_id"], str(_uuid.UUID(d["uuid"])), d["transfer_type"], d["request_type"])


@dataclass
class SchedulerRequirement:
    """protocol.rs:83-92, serde externally-tagged enum:
    {"IterationComplete": i} | {"LayerNameComplete": [name, i]} | {"LayerComplete": [index, i]}."""
    kind: str
    iteration: int
    layer: Optional[object] = None

    def to_json(self):
        return {self.kind: self.iteration} if self.kind == "IterationComplete" else {self.kind: [self.layer, self.iteration]}

    @staticmethod
    def from_json(d) -> "SchedulerRequirement":
        (kind, v), = d.items()
        if kind == "IterationComplete":
            return SchedulerRequirement(kind, int(v))
        if kind in ("LayerNameComplete", "LayerComplete"):
            return SchedulerRequirement(kind, int(v[1]), v[0])
        raise ValueError(f"unknown SchedulerRequirement {kind}")


@dataclass
class LeaderTransferRequest:
    request_id: str
    uuid: str
    requirement: Optional[SchedulerRequirement]
    request_type: str

    def to_json(self) -> dict:
        return {"request_id": self.request_id, "uuid": self.uuid,
                "requirement": self.requirement.to_json() if self.requirement else None, "request_type": self.request_type}

    @staticmethod
    def from_json(d: dict) -> "LeaderTransferRequest":
        req = d.get("requirement")
        return LeaderTransferRequest(d["request_id"], str(_uuid.UUID(d["uuid"])),
                                     SchedulerRequirement.from_json(req) if req is not None else None, d["request_type"])


@dataclass
class BlockTransferRequest:
    """distributed/utils.rs:47-84; `connector_req` is omitted from the JSON when None."""
    from_pool: str
    to_pool: str
    blocks: List[Tuple[int, int]]
    connector_req: Optional[LeaderTransferRequest] = None

    def to_json(self) -> dict:
        d = {"from_pool": self.from_pool, "to_pool": self.to_pool, "blocks": [[int(a), int(b)] for a, b in self.blocks]}
        if self.connector_req is not None:
            d["connector_req"] = self.connector_req.to_json()
        return d

    @staticmethod
    def from_json(d: dict) -> "BlockTransferRequest":
        for k in ("from_pool", "to_pool"):
            if d[k] not in (DEVICE, HOST, DISK):
                raise ValueError(f"unknown pool {d[k]}")
        cr = d.get("connector_req")
        return BlockTransferRequest(d["from_pool"], d["to_pool"], [(int(a), int(b)) for a, b in d["blocks"]],
                                    LeaderTransferRequest.from_json(cr) if cr is not None else None)


@dataclass
class ConnectorMetadata:
    """connector.rs:158-185."""
    iteration: int
    new_slots: List[dict] = field(default_factory=list)            # {request_id, expected_immediate_ops}
    operations: List[WorkerTransferRequest] = field(default_factory=list)

    def create_slot(self, request_id: str, expected_immediate_ops: int) -> None:
        self.new_slots.append({"request_id": request_id, "expected_immediate_ops": int(expected_immediate_ops)})

    def add_operations(self, ops: Iterable[WorkerTransferRequest]) -> None:
        self.operations.extend(ops)

    def to_bytes(self) -> bytes:
        return json.dumps({"iteration": self.iteration, "new_slots": self.new_slots,
                           "operations": [o.to_json() for o in self.operations]}).encode()

    @staticmethod
    def from_bytes(b: bytes) -> "ConnectorMetadata":
        d = json.loads(b)
        return ConnectorMetadata(int(d["iteration"]), [dict(s) for s in d["new_slots"]],
                                 [WorkerTransferRequest.from_json(o) for o in d["operations"]])


# ----------------------------------------------------------------------------------------------- bookkeeping
class _Slot:
    """WorkerSchedulerClientSlot (scheduler.rs:148-177): complete when completed == len(operations)."""

    def __init__(self, expected_immediate_ops: int):
        self.operations: List[str] = []
        self.completed: Set[str] = set()        # uuids whose bytes have landed (a set: a retry can never double-count)
        self.failed: Dict[str, str] = {}        # uuid -> error text of transfers that aborted
        self.expected_immediate_ops = expected_immediate_ops

    def is_complete(self) -> bool:
        return all(u in self.completed or u in self.failed for u in self.operations)


def layer_separate_auto(shape: Sequence[int], num_device_blocks: int) -> BlockDimension:
    """LayoutType::layer_separate_auto (lib/llm/src/block_manager/layout.rs:163-176):
    shape[0] >= num_blocks -> the block dimension comes first, else second (vLLM's [2, num_blocks, ...])."""
    if len(shape) < 2:
        raise ValueError(f"cannot detect layout from shape {list(shape)}")
    return BlockDimension.BlockIsFirstDim if shape[0] >= num_device_blocks else BlockDimension.BlockIsSecondDim


class KvConnectorWorker:
    """`KvConnectorWorker(py_drt, vllm_worker_id)` (worker.rs:479-559).  `drt` is accepted and ignored: the Rust
    runtime is Dynamo's; this object only needs a CUDA device."""

    def __init__(self, drt=None, vllm_worker_id: str = "0", host_blocks: int = 0):
        self.worker_id = vllm_worker_id
        self.mgr: Optional[TransferManager] = None
        self.pools: Dict[str, int] = {}
        self.kv_cache_layers: List[Tuple[str, object]] = []
        self.layer_events: List[int] = []
        self._host_blocks = host_blocks
        self._host_mem = None
        self.slots: Dict[str, _Slot] = {}
        self.bound = False
        self.iteration = 0
        self.worker_iteration = 0
        self.layers_complete = 0
        self.offloading_operations: List[WorkerTransferRequest] = []
        self.maybe_finished_onboarding: Set[str] = set()
        self.maybe_finished_offloading: Set[str] = set()
        self._completed_iterations: Set[int] = set()
        self._completed_layers: Set[Tuple[int, int]] = set()
        self._pending: List[Tuple[BlockTransferRequest, Optional[TransferOptions]]] = []   # waiting for their requirement
        self._inflight: List[Tuple[TransferCompleteNotification, Optional[LeaderTransferRequest]]] = []
        self._enqueued: Dict[Tuple[str, str], int] = {}      # (request_id, uuid) -> epoch at worker-side enqueue
        self._unprocessed: Dict[str, Set[str]] = {}           # request_id -> uuids completed before their slot existed
        self._early: Set[Tuple[str, str]] = set()             # offloads launched (gated) before the last layer was saved
        self.failures: List[Tuple[Optional[str], Optional[str], str]] = []   # transfers that aborted: (request_id, uuid, error)
        self._ready_flags = None
        self._helper_stream = None
        self._epoch = 0

    # -- registration ------------------------------------------------------------------------------------
    def register_kv_caches(self, num_device_blocks: int, page_size: int, device_id: int, dtype_width_bytes: int,
                           kv_caches: Sequence[Tuple[str, object]], raw_event_handles: Sequence[int],
                           device_layout_type=None, host_layout_type=None, disk_layout_type=None,
                           outer_dim: Optional[int] = None, inner_dim: Optional[int] = None) -> None:
        if self.mgr is not None:
            raise RuntimeError("kvbm worker already registered")                    # worker.rs:139-142
        if len(kv_caches) != len(raw_event_handles):
            raise AssertionError("kv_caches and raw_event_handles must have the same length")   # worker.rs:144-148
        self.kv_cache_layers = list(kv_caches)
        self.layer_events = [int(h) for h in raw_event_handles]
        first = kv_caches[0][1]
        shape = list(first.shape)
        block_dim = device_layout_type if isinstance(device_layout_type, BlockDimension) else layer_separate_auto(shape, num_device_blocks)
        if outer_dim is not None and inner_dim is not None:                          # explicit dims: use as they are
            od, inner = outer_dim, inner_dim
        else:
            # distributed/worker.rs:554-578: outer_dim is encoded in the shape when the candidate axis is <= 2
            # ([outer, n_blocks, page, inner] / [n_blocks, outer, page, inner]); otherwise the tensor has no K/V
            # axis (MLA: [n_blocks, page, latent]) -> outer_dim = 1 and inner_dim from every dim after n_blocks
            candidate = shape[1] if block_dim == BlockDimension.BlockIsFirstDim else shape[0]
            tail = shape[2:] if candidate <= 2 else (shape[1:] if block_dim == BlockDimension.BlockIsFirstDim else shape[2:])
            per_block = 1
            for s in tail:
                per_block *= int(s)
            od = outer_dim if outer_dim is not None else (candidate if candidate <= 2 else 1)
            inner = inner_dim if inner_dim is not None else per_block // page_size
        if od not in (1, 2):
            raise ValueError(f"outer_dim must be 1 or 2, got {od}")
        cfg = LayoutConfig(num_device_blocks, len(kv_caches), od, page_size, inner, dtype_width_bytes=dtype_width_bytes,
                           allow_fp8=dtype_width_bytes == 1)
        on_device = bool(getattr(first, "is_cuda", False))
        self.mgr = TransferManager(device=device_id if on_device else -1, worker_id=stable_worker_id(self.worker_id))
        bases = [int(t.data_ptr()) for _, t in kv_caches]
        sizes = [int(t.numel() * t.element_size()) for _, t in kv_caches]
        self.pools[DEVICE] = self.mgr.register_layer_separate(cfg, bases, sizes, block_dim,
                                                              StorageKind.Device if on_device else StorageKind.System, device_id)
        self.device_config = cfg
        if self._host_blocks:
            import torch
            hcfg = LayoutConfig(self._host_blocks, cfg.num_layers, cfg.outer_dim, cfg.page_size, cfg.inner_dim,
                                dtype_width_bytes=cfg.dtype_width_bytes, allow_fp8=cfg.allow_fp8)
            self._host_mem = torch.zeros(hcfg.required_bytes(), dtype=torch.uint8)
            if on_device:
                self._host_mem = self._host_mem.pin_memory()
            # host pool = FullyContiguous, the reference's default host_layout_type (worker.rs:214)
            self.pools[HOST] = self.mgr.register_fully_contiguous(hcfg, self._host_mem.data_ptr(), self._host_mem.numel(),
                                                                  StorageKind.Pinned if on_device else StorageKind.System)
        if on_device:
            import torch
            self._ready_flags = torch.zeros(cfg.num_layers, dtype=torch.int32, device=f"cuda:{device_id}")
            self._helper_stream = torch.cuda.Stream(device=device_id, priority=-1)

    # -- per-iteration protocol --------------------------------------------------------------------------
    def bind_connector_metadata(self, metadata: bytes) -> None:
        md = ConnectorMetadata.from_bytes(metadata)                                   # worker.rs:239
        self.bound = True
        self.iteration = md.iteration
        self.layers_complete = 0
        self.worker_iteration += 1                                                   # connector.start_next_iteration()
        if self.worker_iteration != md.iteration:
            raise AssertionError(f"iteration mismatch: worker {self.worker_iteration} vs metadata {md.iteration}")
        for s in md.new_slots:
            if s["request_id"] in self.slots:
                raise AssertionError("slot already exists")
            self._new_slot(s["request_id"], int(s["expected_immediate_ops"]))        # create_slot_with_immediate_ops
        onboarding, offloading = [], []
        for op in md.operations:
            (onboarding if op.transfer_type == LOAD else offloading).append(op)
        for op in onboarding:                                                        # enqueued immediately
            self._enqueue(op)
            self.maybe_finished_onboarding.add(op.request_id)
        self.offloading_operations = offloading                                      # deferred to the last layer
        self._epoch += 1

    def clear_connector_metadata(self) -> None:
        assert self.bound, "connector metadata not bound"
        self.bound = False
        self._completed_iterations.add(self.worker_iteration)                        # mark_iteration_complete
        self.iteration = 0
        self.layers_complete = 0
        self._run_ready()

    def save_kv_layer(self, layer_name: str, kv_layer=None) -> None:
        self.layers_complete += 1
        idx = self.layers_complete - 1
        if self._ready_flags is not None and idx < len(self.layer_events):
            # device-side: helper stream waits the layer's event, then releases the layer's ready flag (no host block)
            ev = self.layer_events[idx]
            if ev:
                K.check(K.stream_wait_event(int(self._helper_stream.cuda_stream), ev), "stream_wait_event")
            K.check(K.set_flags(self._ready_flags.data_ptr(), idx, 1, self._epoch, int(self._helper_stream.cuda_stream)), "set_flags")
        self._completed_layers.add((idx, self.worker_iteration))
        if self.layers_complete == len(self.kv_cache_layers):
            ops, self.offloading_operations = self.offloading_operations, []
            for op in ops:                                                           # worker.rs:342-350 without the host sync
                self._enqueue(op)
        self._run_ready()

    def get_finished(self, finished_requests: Iterable[str]) -> Tuple[Set[str], Set[str]]:
        """worker.rs:354-470."""
        self._poll()
        for rid in finished_requests:
            if rid not in self.slots:
                continue                                                             # "assuming never started"
            if rid in self.maybe_finished_onboarding or rid in self.maybe_finished_offloading:
                continue
            self.maybe_finished_offloading.add(rid)
        done_off = {r for r in self.maybe_finished_offloading if self.slots[r].is_complete()}
        for r in done_off:
            self.maybe_finished_offloading.discard(r)
            self.slots.pop(r, None)
            self._unprocessed.pop(r, None)
        done_on = {r for r in self.maybe_finished_onboarding if self.slots[r].is_complete()}
        for r in done_on:
            self.maybe_finished_onboarding.discard(r)
            self.slots.pop(r, None)
            self._unprocessed.pop(r, None)
        return done_off, done_on

    # -- transfers issued by the leader -------------------------------------------------------------------
    def handle_block_transfer(self, request, options: Optional[TransferOptions] = None) -> None:
        """A `BlockTransferRequest` (JSON bytes, dict or object) as the leader sends it over ZMQ
        (distributed/transfer.rs:304-395).  Scheduled requests wait for their `SchedulerRequirement`."""
        if isinstance(request, (bytes, str)):
            request = BlockTransferRequest.from_json(json.loads(request))
        elif isinstance(request, dict):
            request = BlockTransferRequest.from_json(request)
        cr = request.connector_req
        if cr is not None and cr.request_type == IMMEDIATE and cr.request_id in self.slots:
            # immediate ops are not announced in the metadata: record them so is_complete() counts them (record_operation)
            slot = self.slots[cr.request_id]
            if cr.uuid not in slot.operations:
                slot.operations.append(cr.uuid)
        self._pending.append((request, options))
        self._run_ready()

    def has_slot(self, request_id: str) -> bool:
        return request_id in self.slots

    def is_complete(self, request_id: str) -> bool:
        self._poll()
        s = self.slots.get(request_id)
        return True if s is None else s.is_complete()

    def ready_flags_ptr(self) -> int:
        return int(self._ready_flags.data_ptr()) if self._ready_flags is not None else 0

    def close(self) -> None:
        if self.mgr is not None:
            self.mgr.close()
            self.mgr = None

    # -- internals ------------------------------------------------------------------------------------------
    def _new_slot(self, request_id: str, expected_immediate_ops: int) -> None:
        slot = _Slot(expected_immediate_ops)
        buffered = self._unprocessed.get(request_id)
        if buffered:                      # add_slot (scheduler.rs:403-437): results that beat the slot are applied to it
            assert len(buffered) <= max(expected_immediate_ops, len(buffered)), "buffered results exceed expected immediate ops"
            slot.completed |= buffered
        self.slots[request_id] = slot

    def _enqueue(self, op: WorkerTransferRequest) -> None:
        if op.request_id not in self.slots:
            raise AssertionError("slot does not exist")                              # scheduler.rs:220-228
        self.slots[op.request_id].operations.append(op.uuid)
        # the worker half of the two-sided hand-shake (scheduler.rs:462-477, try_prepare_controller :539-570): a Scheduled
        # transfer runs only once BOTH this enqueue and the leader's request have arrived.  The epoch at enqueue time is
        # the one this iteration's per-layer ready flags carry.
        self._enqueued.setdefault((op.request_id, op.uuid), self._epoch)

    def _requirement_met(self, req: Optional[SchedulerRequirement]) -> bool:
        if req is None:
            return True
        if req.kind == "IterationComplete":
            return req.iteration in self._completed_iterations
        if req.kind == "LayerComplete":
            return (int(req.layer), req.iteration) in self._completed_layers or req.iteration in self._completed_iterations
        if req.kind == "LayerNameComplete":
            names = [n for n, _ in self.kv_cache_layers]
            idx = names.index(req.layer) if req.layer in names else -1
            return (idx, req.iteration) in self._completed_layers or req.iteration in self._completed_iterations
        return False

    def _run_ready(self) -> None:
        pending, self._pending = self._pending, []
        for i, (req, options) in enumerate(pending):
            cr = req.connector_req
            if cr is not None and cr.request_type == SCHEDULED:
                # scheduler.rs:539-570: wait for the worker-side enqueue of the same uuid (for offloads that is the last
                # save_kv_layer), and for the SchedulerRequirement when the leader attached one
                enq = (cr.request_id, cr.uuid) in self._enqueued
                if not enq and self._ready_flags is not None and req.from_pool == DEVICE and self.bound and \
                        any(op.uuid == cr.uuid and op.request_id == cr.request_id for op in self.offloading_operations):
                    # this path: an offload announced for the iteration that is running can be launched NOW -- the copy is
                    # gated layer by layer on this iteration's ready flags, so it streams behind the forward pass instead
                    # of starting after the last layer.  (It still counts for the slot only once save_kv_layer enqueues it.)
                    self._enqueued[(cr.request_id, cr.uuid)] = self._epoch
                    self._early.add((cr.request_id, cr.uuid))
                    enq = True
                elif not self._requirement_met(cr.requirement):
                    enq = False
                if not enq:
                    self._pending.append((req, options))
                    continue
            try:
                if req.from_pool not in self.pools or req.to_pool not in self.pools:
                    raise KvbmError(8, f"pool {req.from_pool}->{req.to_pool} is not registered on this worker")
                src_ids = [a for a, _ in req.blocks]
                dst_ids = [b for _, b in req.blocks]
                if options is None and req.from_pool == DEVICE and self._ready_flags is not None:
                    # The reference blocks the host on the last layer's event before it enqueues an offload (worker.rs:341).
                    # Here nothing blocks: the copy itself is gated on the per-layer ready flags that save_kv_layer's
                    # helper stream releases behind the forward pass, so device blocks are never read before they are
                    # written.  A request that is not tied to an iteration (no connector_req) reads the current epoch.
                    epoch = self._enqueued.get((cr.request_id, cr.uuid), self._epoch) if cr is not None else self._epoch
                    if epoch > 0:
                        options = TransferOptions(layer_ready_flags=self.ready_flags_ptr(), epoch=epoch)
                note = self.mgr.execute_transfer(self.pools[req.from_pool], src_ids, self.pools[req.to_pool], dst_ids, options)
            except KvbmError as e:
                self._fail(cr, str(e))                       # the request is dropped; everything behind it stays queued
                self._pending.extend(pending[i + 1:])
                raise
            self._inflight.append((note, cr))
        self._poll()

    def _fail(self, cr: Optional[LeaderTransferRequest], why: str) -> None:
        if cr is not None and cr.request_id in self.slots:
            self.slots[cr.request_id].failed[cr.uuid] = why
        self.failures.append((cr.request_id if cr else None, cr.uuid if cr else None, why))

    def _poll(self) -> None:
        """Exception-safe: a transfer that aborted (gate timeout -> rc -2) or whose notification is unknown is dropped from
        the in-flight list, recorded on its slot as failed (so the request can still finish and be cleaned up) and in
        `self.failures`; completions are per-uuid sets, so a retry can never count one twice."""
        rest = []
        for note, cr in self._inflight:
            try:
                done = note.is_complete()
            except KvbmError as e:
                self._fail(cr, str(e))
                continue
            if done:
                if cr is not None and cr.request_id in self.slots:
                    self.slots[cr.request_id].completed.add(cr.uuid)
                elif cr is not None:
                    # an Immediate transfer can finish before the metadata that creates its slot is bound: keep the result
                    # until the slot appears (Scheduler.unprocessed_immediate_results, scheduler.rs:403-437,510-537)
                    self._unprocessed.setdefault(cr.request_id, set()).add(cr.uuid)
            else:
                rest.append((note, cr))
        self._inflight = rest


class TrtllmKvConnectorWorker(KvConnectorWorker):
    """The TRT-LLM flavour of the worker (`PyTrtllmKvConnectorWorker`,
    /root/reference/lib/bindings/kvbm/src/block_manager/vllm/connector/trtllm_worker.rs:31-60,555-645): ONE
    FullyContiguous KV tensor `[num_blocks, num_layers, outer, page, inner...]` (distributed/worker.rs:528-549), method
    names `bind_connector_meta` / `start_load_kv` / `execute_offload_operations` / `save_kv_layer(layer_idx)` /
    `submit_offload_on_event`, loads enqueued by `start_load_kv` instead of at bind time (:371-380)."""

    def __init__(self, drt=None, trtllm_rank: str = "0", host_blocks: int = 0):
        super().__init__(drt, trtllm_rank, host_blocks)
        self.onboarding_operations: List[WorkerTransferRequest] = []

    def register_kv_caches(self, num_device_blocks: int, page_size: int, device_id: int, dtype_width_bytes: int,
                           kv_cache_tensor, raw_event_handles: Sequence[int]) -> None:
        if self.mgr is not None:
            raise RuntimeError("kvbm worker already registered")                    # trtllm_worker.rs:231-234
        shape = [int(x) for x in kv_cache_tensor.shape]
        if len(shape) < 4 or shape[0] < num_device_blocks:
            raise ValueError(f"Unsupported kv cache layout. Got shape: {shape}")   # distributed/worker.rs:517-526
        nl, od = shape[1], shape[2]
        per = 1
        for x in shape[3:]:
            per *= x
        cfg = LayoutConfig(num_device_blocks, nl, od, page_size, per // page_size, dtype_width_bytes=dtype_width_bytes,
                           allow_fp8=dtype_width_bytes == 1)
        on_device = bool(getattr(kv_cache_tensor, "is_cuda", False))
        self.mgr = TransferManager(device=device_id if on_device else -1, worker_id=stable_worker_id(self.worker_id))
        self.kv_cache_layers = [(f"layer_{l}", kv_cache_tensor) for l in range(nl)]
        self.layer_events = [int(h) for h in raw_event_handles]
        self.pools[DEVICE] = self.mgr.register_fully_contiguous(
            cfg, int(kv_cache_tensor.data_ptr()), int(kv_cache_tensor.numel() * kv_cache_tensor.element_size()),
            StorageKind.Device if on_device else StorageKind.System, device_id)
        self.device_config = cfg
        if self._host_blocks:
            import torch
            hcfg = LayoutConfig(self._host_blocks, nl, od, page_size, cfg.inner_dim, dtype_width_bytes=dtype_width_bytes,
                                allow_fp8=cfg.allow_fp8)
            self._host_mem = torch.zeros(hcfg.required_bytes(), dtype=torch.uint8)
            if on_device:
                self._host_mem = self._host_mem.pin_memory()
            self.pools[HOST] = self.mgr.register_fully_contiguous(hcfg, self._host_mem.data_ptr(), self._host_mem.numel(),
                                                                  StorageKind.Pinned if on_device else StorageKind.System)
        if on_device:
            import torch
            self._ready_flags = torch.zeros(nl, dtype=torch.int32, device=f"cuda:{device_id}")
            self._helper_stream = torch.cuda.Stream(device=device_id, priority=-1)

    def bind_connector_meta(self, metadata: bytes) -> None:
        """trtllm_worker.rs:282-346: like the vLLM bind, but loads are only recorded here and enqueued by start_load_kv."""
        md = ConnectorMetadata.from_bytes(metadata)
        self.bound = True
        self.iteration = md.iteration
        self.layers_complete = 0
        self.worker_iteration += 1
        if self.worker_iteration != md.iteration:
            raise AssertionError(f"iteration mismatch: worker {self.worker_iteration} vs metadata {md.iteration}")
        for sl in md.new_slots:
            if sl["request_id"] in self.slots:
                raise AssertionError("slot already exists")
            self._new_slot(sl["request_id"], int(sl["expected_immediate_ops"]))
        self.onboarding_operations = [op for op in md.operations if op.transfer_type == LOAD]
        self.offloading_operations = [op for op in md.operations if op.transfer_type == STORE]
        self._epoch += 1

    bind_connector_metadata = bind_connector_meta

    def start_load_kv(self) -> None:
        for op in self.onboarding_operations:                                        # :371-380 (the list is cloned, not taken)
            self._enqueue(op)
            self.maybe_finished_onboarding.add(op.request_id)

    def execute_offload_operations(self) -> None:
        ops, self.offloading_operations = self.offloading_operations, []
        for op in ops:
            self._enqueue(op)
        self._run_ready()

    def save_kv_layer(self, layer_idx: int, kv_layer=None) -> None:                  # :357-369; the index is ignored there too
        super().save_kv_layer(f"layer_{self.layers_complete}", kv_layer)

    def submit_offload_on_event(self, event: int) -> None:
        """:526-553: the offload is tied to ONE event instead of per-layer calls.  Here the helper stream waits that event
        and releases every layer's ready flag, then the stores are enqueued -- still without blocking the host."""
        if self._ready_flags is not None:
            if event:
                K.check(K.stream_wait_event(int(self._helper_stream.cuda_stream), int(event)), "stream_wait_event")
            K.check(K.set_flags(self._ready_flags.data_ptr(), 0, len(self.kv_cache_layers), self._epoch,
                                int(self._helper_stream.cuda_stream)), "set_flags")
        for l in range(len(self.kv_cache_layers)):
            self._completed_layers.add((l, self.worker_iteration))
        self.layers_complete = len(self.kv_cache_layers)
        self.execute_offload_operations()
