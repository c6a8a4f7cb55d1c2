"""Leader (scheduler) side of Dynamo's KVBM connector (SURVEY.md §8 f1), the half that PRODUCES what
`connector.KvConnectorWorker` consumes.

Mirrors, relative to /root/reference/lib/bindings/kvbm/src/block_manager/vllm/:
  connector/leader.rs:47-77      trait Leader {get_num_new_matched_tokens, update_state_after_alloc,
                                 build_connector_metadata, request_finished, has_slot, create_slot}
  connector/leader.rs:199-600    KvConnectorLeader: iteration counter, inflight / onboarding sets, the three loops of
                                 build_connector_metadata (onboarding slots, new requests, cached requests) and the
                                 "unscheduled -> skipped" pass
  connector/leader/slot.rs:63-96       SlotState
  connector/leader/slot.rs:593-896     apply_scheduler_output: device-block suffix/prefix overlap contract, candidate
                                       blocks = full blocks between `evaluated_blocks` and the new position, contiguous
                                       priority filter that TERMINATES offloading at the first block below the threshold
  connector/leader/slot.rs:977-1126    acquire_local_matches: host match after the device-computed prefix; a match that
                                       would cover the whole prompt drops its last block (one token must be computed)
  connector/leader/slot.rs:1128-1196   trigger_onboarding
  connector/leader/slot.rs:1246-1341   offload_blocks -> WorkerTransferRequest{Store, Scheduled} + transfer-engine request,
                                       onboard_blocks -> WorkerTransferRequest{Load, Immediate}; both share one uuid
  connector.rs:21-110                  SchedulerOutput / NewRequestData / CachedRequestData
The transfer-engine half (slot.rs:1442-1820: allocate host blocks, send a `BlockTransferRequest` to the workers, register
the blocks once the copy is done) is the small `HostPool` + `send` callback below; the bytes themselves move through
`KvConnectorWorker.handle_block_transfer` -> `TransferManager` -> the sm_90a kernels.  Dynamo's block manager (pools with
reuse policies, disk tier, metrics, ZMQ) stays Dynamo's: this class is what makes the worker's protocol drivable end to end.
"""
from __future__ import annotations

import uuid as _uuid
from collections import OrderedDict
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Sequence, Set, Tuple

from . import router as _router
from .connector import (DEVICE, HOST, IMMEDIATE, LOAD, SCHEDULED, STORE, BlockTransferRequest, ConnectorMetadata,
                        LeaderTransferRequest, WorkerTransferRequest)

# SlotState (slot.rs:63-96); OnboardStaged / Onboarding carry a token count
INITIALIZED, ONBOARD_STAGED, ONBOARDING, PREFILLING, SKIPPED_PREFILL = "Initialized", "OnboardStaged", "Onboarding", "Prefilling", "SkippedPrefill"
DECODING, SKIPPED_DECODE, FINISHING, FINISHED, PREEMPTED = "Decoding", "SkippedDecode", "Finishing", "Finished", "Preempted"


class SlotError(RuntimeError):
    pass


@dataclass
class KvbmRequest:
    """vllm/request.rs: what create_slot receives besides the tokens."""
    request_id: str
    lora_name: Optional[str] = None
    salt_hash: int = 0


@dataclass
class NewRequestData:
    request_id: str
    prompt_token_ids: List[int]
    block_ids: List[int]
    num_computed_tokens: int
    priorities: Optional[List[int]] = None


@dataclass
class CachedRequestData:
    request_id: str
    resumed_from_preemption: bool
    new_token_ids: List[int]
    new_block_ids: List[int]
    num_computed_tokens: int
    priorities: Optional[List[int]] = None


@dataclass
class SchedulerOutput:
    """connector.rs:21-110."""
    new_requests: List[NewRequestData] = field(default_factory=list)
    cached_requests: List[CachedRequestData] = field(default_factory=list)
    num_scheduled_tokens: Dict[str, int] = field(default_factory=dict)

    def add_new_request(self, request_id, prompt_token_ids, block_ids, num_computed_tokens, priorities=None):
        self.new_requests.append(NewRequestData(request_id, list(prompt_token_ids), list(block_ids), num_computed_tokens, priorities))

    def add_cached_request(self, request_id, resumed_from_preemption, new_token_ids, new_block_ids, num_computed_tokens, priorities=None):
        self.cached_requests.append(CachedRequestData(request_id, resumed_from_preemption, list(new_token_ids), list(new_block_ids),
                                                      num_computed_tokens, priorities))

    def add_num_scheduled_tokens(self, mapping: Dict[str, int]):
        self.num_scheduled_tokens.update(mapping)


class HostPool:
    """The host tier as the leader sees it: free blocks, and registered (immutable, matchable) blocks keyed by sequence
    hash with least-recently-used reuse -- the role of `block_manager.host()` in slot.rs (match_sequence_hashes_blocking,
    allocate_blocks_blocking, register_blocks)."""

    def __init__(self, num_blocks: int):
        self.num_blocks = num_blocks
        self.free: List[int] = list(range(num_blocks - 1, -1, -1))
        self.registered: "OrderedDict[int, int]" = OrderedDict()     # sequence hash -> host block id (LRU order)
        self.in_flight: Set[int] = set()                              # allocated, copy not finished yet

    def match_sequence_hashes(self, hashes: Sequence[int]) -> List[int]:
        out = []
        for h in hashes:
            b = self.registered.get(h)
            if b is None:
                break
            self.registered.move_to_end(h)
            out.append(b)
        return out

    def allocate(self, n: int) -> Optional[List[int]]:
        while len(self.free) < n and self.registered:
            _, b = self.registered.popitem(last=False)                # evict the least recently used registered block
            self.free.append(b)
        if len(self.free) < n:
            return None
        got = [self.free.pop() for _ in range(n)]
        self.in_flight.update(got)
        return got

    def register(self, hashes: Sequence[int], blocks: Sequence[int]) -> None:
        for h, b in zip(hashes, blocks):
            self.in_flight.discard(b)
            old = self.registered.pop(h, None)
            if old is not None and old != b:
                self.free.append(old)
            self.registered[h] = b

    def release(self, blocks: Sequence[int]) -> None:
        for b in blocks:
            if b in self.in_flight:
                self.in_flight.discard(b)
                self.free.append(b)


class _Slot:
    """VllmConnectorSlot (slot.rs:323-520)."""

    def __init__(self, request_id: str, tokens: Sequence[int], block_size: int, lora_name: Optional[str], salt_hash: int,
                 leader: "KvConnectorLeader"):
        self.request_id = request_id
        self.block_size = block_size
        self.lora_name = lora_name
        self.salt_hash = salt_hash
        self.leader = leader
        self.tokens: List[int] = list(tokens)
        self.state = INITIALIZED
        self.state_tokens = 0
        self.current_position = 0
        self.evaluated_blocks = 0
        self.device_blocks: List[int] = []
        self.pending_operations: Optional[List[WorkerTransferRequest]] = None
        self.staging_from_host: Optional[List[int]] = None
        self.stored_block_priorities: Dict[int, int] = {}
        self.offload_terminated_at_block: Optional[int] = None
        self.iteration_first_scheduled: Optional[int] = None
        self.tokens_cached_from_device = self.tokens_cached_from_host = 0
        self.outstanding: Set[str] = set()            # uuids of transfers the engine has not reported complete
        self._hash_cache: Tuple[int, List[int]] = (0, [])

    # TokenBlockSequence: only FULL blocks have hashes (lib/llm/src/tokens.rs); the chain uses the router's XXH3 scheme
    def sequence_hashes(self) -> List[int]:
        n_full = len(self.tokens) // self.block_size
        if self._hash_cache[0] != n_full:
            local = _router.compute_block_hash_for_seq(self.tokens[:n_full * self.block_size], self.block_size, self.lora_name)
            if self.salt_hash and local:
                local[0] ^= self.salt_hash & 0xFFFFFFFFFFFFFFFF      # the salt separates otherwise identical prefixes
            self._hash_cache = (n_full, _router.compute_seq_hash_for_block(local))
        return self._hash_cache[1]

    def total_tokens(self) -> int:
        return len(self.tokens)

    def mark_as_skipped(self) -> None:                                   # slot.rs:484-520
        if self.state == PREFILLING:
            self.state = SKIPPED_PREFILL
        elif self.state == DECODING:
            self.state = SKIPPED_DECODE

    def take_pending_operations(self) -> Optional[List[WorkerTransferRequest]]:
        ops, self.pending_operations = self.pending_operations, None
        return ops

    def _append_pending(self, op: WorkerTransferRequest) -> None:
        if self.pending_operations is None:
            self.pending_operations = []
        self.pending_operations.append(op)

    # -- slot.rs:977-1126 ---------------------------------------------------------------------------------------
    def acquire_local_matches(self, num_computed_tokens: int) -> None:
        if self.state == ONBOARD_STAGED:
            return
        if self.state not in (INITIALIZED, PREEMPTED):
            raise SlotError(f"slot must be in the NotScheduled or Preempted state to acquire local matches; got {self.state}")
        bs = self.block_size
        hashes = self.sequence_hashes()
        lookup = hashes[num_computed_tokens // bs:]
        if not lookup:
            return
        host_blocks = self.leader.host.match_sequence_hashes(lookup)
        self.tokens_cached_from_host = len(host_blocks) * bs
        if not host_blocks:
            return
        new_tokens = len(host_blocks) * bs
        if num_computed_tokens + new_tokens == self.total_tokens():      # on a block boundary: keep one block to compute
            host_blocks.pop()
            new_tokens -= bs
        if new_tokens == 0:
            return
        self.staging_from_host = host_blocks
        self.state, self.state_tokens = ONBOARD_STAGED, new_tokens

    # -- slot.rs:1128-1196 --------------------------------------------------------------------------------------
    def trigger_onboarding(self, num_external_tokens: int) -> None:
        if self.state != ONBOARD_STAGED:
            raise SlotError(f"slot must be in the OnboardStaged state to trigger onboarding; got {self.state}")
        assert self.evaluated_blocks == 0 and self.current_position % self.block_size == 0
        self.evaluated_blocks = self.current_position // self.block_size
        host_blocks, self.staging_from_host = self.staging_from_host, None
        if host_blocks:
            dst = self.device_blocks[self.evaluated_blocks:self.evaluated_blocks + len(host_blocks)]
            assert len(dst) == len(host_blocks)
            self._onboard_blocks(host_blocks, dst)
            self.evaluated_blocks += len(host_blocks)
        self.state, self.state_tokens = ONBOARDING, num_external_tokens
        self.advance_computed_position(num_external_tokens)

    def advance_computed_position(self, n: int) -> None:                 # slot.rs:1204-1223
        if self.current_position + n > self.total_tokens():
            raise SlotError(f"cannot advance computed position from {self.current_position} by {n} tokens, total tokens is {self.total_tokens()}")
        self.current_position += n

    # -- slot.rs:593-896 ----------------------------------------------------------------------------------------
    def apply_scheduler_output(self, tokens: Sequence[int], block_ids: Sequence[int], num_computed_tokens: int,
                               num_scheduled_tokens: int, priorities: Optional[Sequence[int]] = None) -> None:
        if priorities is not None:
            assert len(priorities) == len(block_ids), "priorities length must match block_ids length"
        if tokens:
            self.state = DECODING
            self.tokens.extend(int(t) for t in tokens)
        else:
            self.state = PREFILLING
        bs = self.block_size
        self.current_position = max(self.current_position, num_computed_tokens)
        self.evaluated_blocks = max(self.evaluated_blocks, num_computed_tokens // bs)
        if block_ids:
            block_ids = list(block_ids)
            overlap = 0
            if block_ids[0] in self.device_blocks:
                pos = len(self.device_blocks) - 1 - self.device_blocks[::-1].index(block_ids[0])
                suffix = len(self.device_blocks) - pos
                assert suffix <= len(block_ids) and self.device_blocks[pos:] == block_ids[:suffix], \
                    f"device_blocks contract violation: block_ids[0]={block_ids[0]} found at device_blocks[{pos}] but the suffix does not match"
                overlap = suffix
            new_ids = block_ids[overlap:]
            existing = set(self.device_blocks)
            for b in new_ids:
                assert b not in existing, f"device_blocks contract violation: block {b} already in device_blocks"
            self.device_blocks.extend(new_ids)
        if priorities is not None:
            for b, p in zip(block_ids, priorities):
                self.stored_block_priorities[b] = int(p)
        if self.offload_terminated_at_block is not None:
            self.current_position += num_scheduled_tokens
            return
        next_position = self.current_position + num_scheduled_tokens
        assert next_position <= len(self.device_blocks) * bs, \
            f"next_position: {next_position} > device_blocks.len() {len(self.device_blocks)} * block_size {bs}"
        if next_position > self.total_tokens():                          # the engine stopped providing tokens
            self.state = DECODING
            return
        num_candidate = next_position // bs - self.evaluated_blocks
        if num_candidate > 0:
            cand = self.device_blocks[self.evaluated_blocks:self.evaluated_blocks + num_candidate]
            assert len(cand) == num_candidate, "device block overflow"
            prios = [self.stored_block_priorities.get(b, 0) for b in cand]
            thr = self.leader.offload_min_priority
            n_off = num_candidate
            if thr > 0:
                n_off = 0
                for p in prios:
                    if p < thr:
                        break
                    n_off += 1
            if n_off > 0:
                hashes = self.sequence_hashes()[self.evaluated_blocks:self.evaluated_blocks + n_off]
                self._offload_blocks(cand[:n_off], hashes, prios[:n_off])
            if n_off < num_candidate:                                     # a gap would break contiguity: stop for good
                self.offload_terminated_at_block = self.evaluated_blocks + n_off
            self.evaluated_blocks += num_candidate
        self.current_position += num_scheduled_tokens

    def mark_as_finished(self) -> None:                                  # slot.rs:905-958
        self.state = FINISHING if (self.pending_operations or self.outstanding) else FINISHED

    def reset_after_preemption(self) -> None:                            # slot.rs:543-560
        self.state = PREEMPTED
        self.current_position = 0
        self.evaluated_blocks = 0
        self.device_blocks = []
        self.iteration_first_scheduled = None
        self.offload_terminated_at_block = None

    # -- slot.rs:1246-1341: engine request + worker request share one uuid ---------------------------------------
    def _offload_blocks(self, block_ids: Sequence[int], seq_hashes: Sequence[int], priorities: Sequence[int]) -> None:
        if self.state in (FINISHING, FINISHED):
            return
        assert len(block_ids) == len(seq_hashes) == len(priorities)
        op = str(_uuid.uuid4())
        self.leader._engine_offload(self, op, list(block_ids), list(seq_hashes))
        self._append_pending(WorkerTransferRequest(self.request_id, op, STORE, SCHEDULED))

    def _onboard_blocks(self, host_blocks: Sequence[int], dst_block_ids: Sequence[int]) -> None:
        op = str(_uuid.uuid4())
        self.leader._engine_onboard(self, op, list(host_blocks), list(dst_block_ids))
        self._append_pending(WorkerTransferRequest(self.request_id, op, LOAD, IMMEDIATE))


class KvConnectorLeader:
    """`KvConnectorLeader(worker_id, drt, page_size, leader)` (leader.rs:91-197).  `send(BlockTransferRequest)` delivers a
    transfer request to the worker(s) -- ZMQ in Dynamo (distributed/transfer.rs:304-395), a direct call in one process."""

    def __init__(self, worker_id: str, page_size: int, host_blocks: int, send: Callable[[BlockTransferRequest], None],
                 offload_min_priority: int = 0, drt=None):
        self.worker_id = worker_id
        self.block_size = page_size
        self.host = HostPool(host_blocks)
        self.send = send
        self.offload_min_priority = offload_min_priority
        self.slots: Dict[str, _Slot] = {}
        self.inflight_requests: Set[str] = set()
        self.onboarding_slots: Set[str] = set()
        self.iteration_counter = 0
        self.matched_tokens = 0                                          # kvbm_metrics.matched_tokens
        self._ops: Dict[str, Tuple[str, str, List[int], List[int]]] = {}  # uuid -> (request_id, kind, hashes, host blocks)

    # -- trait Leader --------------------------------------------------------------------------------------------
    def create_slot(self, request: KvbmRequest, tokens: Sequence[int]) -> None:
        if request.request_id in self.slots:
            raise SlotError(f"slot {request.request_id} already exists")
        self.slots[request.request_id] = _Slot(request.request_id, tokens, self.block_size, request.lora_name, request.salt_hash, self)
        self.inflight_requests.add(request.request_id)

    def has_slot(self, request_id: str) -> bool:
        return request_id in self.slots

    def _slot(self, request_id: str) -> _Slot:
        s = self.slots.get(request_id)
        if s is None:
            raise SlotError(f"slot not found: {request_id}")
        return s

    def get_num_new_matched_tokens(self, request_id: str, request_num_tokens: int, num_computed_tokens: int) -> Tuple[int, bool]:
        """leader.rs:216-283.  (0, False) when nothing matches; (n, True) when n external tokens will be onboarded."""
        slot = self._slot(request_id)
        if slot.state == SKIPPED_PREFILL:
            slot.state = PREFILLING
            return 0, False
        if slot.state == SKIPPED_DECODE:
            slot.state = DECODING
            return 0, False
        if slot.total_tokens() - num_computed_tokens < self.block_size:
            return 0, False
        slot.acquire_local_matches(num_computed_tokens)
        if slot.state == ONBOARD_STAGED:
            self.matched_tokens += slot.state_tokens
            return slot.state_tokens, True
        return 0, False

    def update_state_after_alloc(self, request_id: str, block_ids: Sequence[int], num_external_tokens: int) -> None:
        """leader.rs:287-327."""
        slot = self._slot(request_id)
        slot.device_blocks.extend(int(b) for b in block_ids)            # append_mutable_device_blocks
        if num_external_tokens > 0:
            num_computed = len(block_ids) * self.block_size - num_external_tokens
            slot.tokens_cached_from_device = num_computed
            slot.advance_computed_position(num_computed)
            slot.trigger_onboarding(num_external_tokens)
            self.onboarding_slots.add(request_id)

    def build_connector_metadata(self, out: SchedulerOutput) -> bytes:
        """leader.rs:329-538."""
        self.iteration_counter += 1
        it = self.iteration_counter
        inflight = set(self.inflight_requests)
        md = ConnectorMetadata(it)
        onboarding, self.onboarding_slots = self.onboarding_slots, set()

        def emit(slot: _Slot, rid: str) -> None:
            ops = slot.take_pending_operations()
            if ops:
                md.create_slot(rid, sum(1 for o in ops if o.request_type == IMMEDIATE))
                md.add_operations(ops)
            else:
                md.create_slot(rid, 0)

        for rid in onboarding:
            emit(self._slot(rid), rid)
            assert rid in inflight, f"request_id {rid} not found in inflight_requests"
            inflight.discard(rid)
        for req in out.new_requests:
            rid = req.request_id
            assert rid in inflight, f"request_id {rid} not found in inflight_requests"
            inflight.discard(rid)
            if any(s["request_id"] == rid for s in md.new_slots):
                continue
            slot = self._slot(rid)
            if slot.iteration_first_scheduled is None:
                slot.iteration_first_scheduled = it
            assert slot.state in (INITIALIZED, ONBOARDING), f"current slot state: {slot.state}"
            slot.apply_scheduler_output([], [], req.num_computed_tokens, out.num_scheduled_tokens.get(rid, 0), None)
            emit(slot, rid)
        for req in out.cached_requests:
            rid = req.request_id
            slot = self._slot(rid)
            if req.resumed_from_preemption:
                slot.reset_after_preemption()
            assert rid in inflight, f"request_id {rid} not found in inflight_requests"
            inflight.discard(rid)
            slot.apply_scheduler_output(req.new_token_ids, req.new_block_ids, req.num_computed_tokens,
                                        out.num_scheduled_tokens.get(rid, 0), req.priorities)
            ops = slot.take_pending_operations()
            if ops:
                md.add_operations(ops)
        for rid in inflight:                                             # in flight but not scheduled this iteration
            self._slot(rid).mark_as_skipped()
        return md.to_bytes()

    def request_finished(self, request_id: str, block_ids: Sequence[int]) -> bool:
        """leader.rs:540-598: False only for an unknown request; True otherwise (the worker reports the real completion)."""
        if request_id not in self.slots:
            self.inflight_requests.discard(request_id)
            return False
        slot = self.slots[request_id]
        slot.mark_as_finished()
        self.inflight_requests.discard(request_id)
        if slot.state == FINISHED:
            del self.slots[request_id]
        return True

    # -- the transfer-engine half (slot.rs:1442-1820) ------------------------------------------------------------
    def _engine_offload(self, slot: _Slot, op: str, device_blocks: List[int], seq_hashes: List[int]) -> None:
        # blocks whose content the host tier already holds are not copied again
        todo = [(b, h) for b, h in zip(device_blocks, seq_hashes) if h not in self.host.registered]
        host = self.host.allocate(len(todo)) if todo else []
        if host is None:                                                  # host tier exhausted by in-flight copies: skip this batch
            todo, host = [], []
        self._ops[op] = (slot.request_id, STORE, [h for _, h in todo], list(host))
        slot.outstanding.add(op)
        self.send(BlockTransferRequest(DEVICE, HOST, [(b, hb) for (b, _), hb in zip(todo, host)],
                                       LeaderTransferRequest(slot.request_id, op, None, SCHEDULED)))

    def _engine_onboard(self, slot: _Slot, op: str, host_blocks: List[int], device_blocks: List[int]) -> None:
        self._ops[op] = (slot.request_id, LOAD, [], list(host_blocks))
        slot.outstanding.add(op)
        self.send(BlockTransferRequest(HOST, DEVICE, list(zip(host_blocks, device_blocks)),
                                       LeaderTransferRequest(slot.request_id, op, None, IMMEDIATE)))

    def transfer_complete(self, op_uuid: str, ok: bool = True) -> None:
        """The worker reported the transfer with this uuid complete (the reply the reference's transfer task awaits,
        slot.rs:1647-1760): offloaded blocks become matchable, a finishing slot may now finish."""
        rec = self._ops.pop(op_uuid, None)
        if rec is None:
            return
        rid, kind, hashes, host = rec
        if kind == STORE:
            if ok:
                self.host.register(hashes, host)
            else:
                self.host.release(host)
        slot = self.slots.get(rid)
        if slot is not None:
            slot.outstanding.discard(op_uuid)
            if slot.state == FINISHING and not slot.outstanding and not slot.pending_operations:
                slot.state = FINISHED
                del self.slots[rid]
