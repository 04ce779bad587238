"""Process-group helpers for shard replication (API mirror of reference ``local/replication/group_utils.py``).

``GroupWrapper`` keeps the reference's method set.  The data-moving methods are rebuilt around the packed
staging buffer of the snapshot engine:

* ``all_gather_batch`` (reference ``:342-375``: for every rank, for every tensor, one ``dist.broadcast`` plus one
  ``.to("cpu")``) -> the local tensors are packed by one kernel straight into this rank's slice of an exchange
  buffer, ONE ``all_gather_into_tensor`` moves all payloads over NVLink, one side-stream drain lands the whole
  buffer in a pinned host slot, and the returned tensors are views of that slot.
* ``isend_state_dict`` / ``irecv_state_dict`` (reference ``:378-449``: one ``dist.send`` / ``dist.recv`` per tensor
  with ``.cuda()`` / ``.cpu()`` bounces) -> one packed send / recv and one scatter kernel.

Host tensors on a CPU backend (gloo) follow the same shape -- flatten, one collective, views -- with plain
host copies; that is not a fallback of the CUDA path: CUDA tensors always go through ``libnvrx_snap.so``.
"""

from __future__ import annotations

import logging
import typing
from dataclasses import dataclass, field
from itertools import islice
from typing import Dict, List, Optional, Tuple, TypeVar, Union

import torch
import torch.distributed as dist

from ...utils import debug_msg, debug_time
from ..base_state_dict import TensorAwareStateDict
from ._torch_future import recv_object_list, send_object_list
from .torch_device_utils import TensorPlaceholder

T = TypeVar("T")
logger = logging.getLogger(__name__)

_HOST_ALIGN = 512


@dataclass(frozen=True)
class ExchangePlanEntry:
    """``sender`` (global rank) ships the state dict ``id_`` to ``receiver`` (global rank)."""

    sender: int
    receiver: int
    id_: str


@dataclass
class ExchangePlan:
    """Ordered list of shard transfers inside ``group``; every rank holds the same plan."""

    group: "GroupWrapper"
    _entries: List[ExchangePlanEntry] = field(default_factory=list)

    def plan(self, *args, **kwargs):
        """Append a transfer (arguments of :class:`ExchangePlanEntry`)."""
        self._entries.append(ExchangePlanEntry(*args, **kwargs))

    @property
    def entries(self) -> Tuple[ExchangePlanEntry]:
        return tuple(self._entries)

    def required_ids(self, rank=None):
        """Ids ``rank`` (default: this rank) has to provide as a sender."""
        if rank is None:
            rank = self.group.get_global_rank()
        return {e.id_ for e in self._entries if e.sender == rank}


def batched(iterable, n):
    """Tuples of ``n`` consecutive items; the last one may be shorter (``itertools.batched`` of 3.12)."""
    if n < 1:
        raise ValueError("n must be at least one")
    it = iter(iterable)
    while chunk := tuple(islice(it, n)):
        yield chunk


def parse_group_sequence(replication_jump, replication_factor, world_size):
    """Replication cliques: ranks ``n, n+J, ..., n+(F-1)J`` for every admissible ``n`` (``J`` = jump, ``F`` = factor).

    Returns the sorted list of rank tuples; ``world_size`` must be a multiple of ``J*F``
    (reference ``:120-146``; docstring example ``strategies.py:215-220``: W=32, J=8, F=2 -> (0,8), (1,9), ...)."""
    assert replication_jump > 0, "Rank cannot store a replica of itself!"
    assert replication_factor > 0, "Tried to create empty replication groups!"
    assert world_size % (replication_jump * replication_factor) == 0, (
        f"Cannot split {world_size} ranks into replication groups! "
        f"Ranks {replication_jump - 1}, {2 * replication_jump - 1}, ... contains "
        f"{world_size // replication_jump} ranks, but this cannot be split into "
        f"groups of size {replication_factor}."
    )
    groups = []
    for residue in range(replication_jump):
        groups.extend(batched(range(residue, world_size, replication_jump), replication_factor))
    groups.sort()
    return groups


# --------------------------------------------------------------------------------------------------
# flat host payloads (CPU backend)
# --------------------------------------------------------------------------------------------------
def _host_layout(nbytes: List[int]) -> Tuple[List[int], int]:
    offs, cur = [], 0
    for nb in nbytes:
        cur = (cur + _HOST_ALIGN - 1) // _HOST_ALIGN * _HOST_ALIGN
        offs.append(cur)
        cur += nb
    return offs, (cur + _HOST_ALIGN - 1) // _HOST_ALIGN * _HOST_ALIGN


def _flatten_host(tensors: List[torch.Tensor], offs: List[int], total: int) -> torch.Tensor:
    flat = torch.zeros(max(total, 1), dtype=torch.uint8)
    for t, off in zip(tensors, offs):
        nb = t.numel() * t.element_size()
        if nb:
            flat[off : off + nb] = t.detach().contiguous().view(-1).view(torch.uint8)
    return flat


def _views_from_flat(flat: torch.Tensor, placeholders: List[TensorPlaceholder], offs: List[int]) -> List[torch.Tensor]:
    """Typed tensors over slices of a flat host buffer, each with a storage of its own (``torch.save`` rejects
    differently typed views of one storage)."""
    raw = flat.numpy()
    out = []
    for tp, off in zip(placeholders, offs):
        meta = tp.hollow_tensor
        if tp.nbytes == 0:
            out.append(torch.empty(meta.shape, dtype=meta.dtype))
        else:
            out.append(torch.frombuffer(raw[off : off + tp.nbytes], dtype=meta.dtype).view(meta.shape))
    return out


class GroupWrapper:
    """A process group (``None`` = the world) with rank translation and the collectives replication needs."""

    def __init__(self, group=None):
        self._group = group
        self.last_snapshots: list = []  # engine Snapshot handles produced by the last all_gather_batch

    @staticmethod
    def wrap(group: "ProcessGroupLike"):
        """``GroupWrapper`` for a ``ProcessGroup``; wrappers pass through."""
        if isinstance(group, GroupWrapper):
            return group
        if isinstance(group, dist.ProcessGroup):
            return GroupWrapper(group)
        raise ValueError(f"Unsupported type: {type(group)}!")

    @staticmethod
    def from_list_of_groups(list_of_groups: List[dist.ProcessGroup]) -> "GroupWrapper":
        """The one group of ``list_of_groups`` this rank belongs to."""
        me = dist.get_rank()
        mine = [g for g in list_of_groups if me in dist.get_process_group_ranks(g)]
        assert len(mine) <= 1, f"Rank {me} is in more groups than one! Groups: {mine}"
        assert len(mine) >= 1, f"Rank {me} not in any process group!"
        return GroupWrapper(mine[0])

    # ---- introspection ------------------------------------------------------------------------
    @property
    def group(self):
        return self._group

    @property
    def backend(self):
        return dist.get_backend(self.group)

    @property
    def supported_devices(self):
        return [torch.device(d) for d in dist.Backend.backend_capability[self.backend]]

    def get_device(self, wanted_device=None):
        """A device the backend can communicate from (``wanted_device`` is validated when given)."""
        if wanted_device is None:
            wanted_device = self.supported_devices[0]
        assert (
            torch.device(wanted_device) in self.supported_devices
        ), f"Selected backend {self.backend} does not support the selected device {wanted_device}!"
        return wanted_device

    def get_group_rank(self, global_rank=None):
        if global_rank is None:
            return dist.get_rank(self.group)
        if self.group is None:
            return global_rank
        return dist.get_group_rank(self.group, global_rank)

    @property
    def my_group_rank(self):
        return self.get_group_rank(None)

    def get_global_rank(self, group_rank=None):
        if group_rank is None or self.group is None:
            return dist.get_rank()
        return dist.get_global_rank(self.group, group_rank)

    @property
    def my_global_rank(self):
        return self.get_global_rank(None)

    @property
    def ranks(self):
        """Global ranks of the members, in group-rank order."""
        if self.group is None:
            return range(dist.get_world_size())
        return dist.get_process_group_ranks(self.group)

    @property
    def world_size(self):
        return dist.get_world_size(self.group)

    def __repr__(self):
        return f"<ProcessGroup of size {self.world_size}, rank: local={self.my_group_rank}, global={self.my_global_rank}>"

    # ---- object collectives -------------------------------------------------------------------
    def all_gather_object(self, my_obj: T) -> List[T]:
        gathered: List[Optional[T]] = [None] * self.world_size
        dist.all_gather_object(gathered, my_obj, group=self.group)
        return typing.cast(List[T], gathered)

    def broadcast(self, *args, **kwargs):
        return dist.broadcast(*args, **kwargs, group=self.group)

    def recv_object(self, src):
        box = [None]
        recv_object_list(box, src, group=self.group)
        return box[0]

    def send_object(self, obj, dst):
        send_object_list([obj], dst, group=self.group)

    # ---- payload collectives ------------------------------------------------------------------
    def all_gather_batch(self, my_tensors: List[torch.Tensor], target_device=None) -> List[List[torch.Tensor]]:
        """All-gather a *list* of tensors: returns, per group rank, that rank's tensors (own rank included).

        CUDA tensors: packed exchange through the snapshot engine; with ``target_device="cpu"`` the result
        tensors are views of a pinned host slot that become valid when the drain finishes (the handles are
        left in ``self.last_snapshots``; wait / release them as for any snapshot)."""
        device_kinds = sorted({t.device.type for t in my_tensors})
        debug_msg(f"tensor_devices={device_kinds}")
        debug_msg(f"{target_device=}")
        with debug_time("all_gather_placeholders"):
            all_placeholders = self._gather_placeholders(my_tensors)
        self.last_snapshots = []
        if any(t.is_cuda for t in my_tensors):
            assert all(t.is_cuda for t in my_tensors), "all_gather_batch: mixed CPU/CUDA tensor lists are not supported"
            from ...b200.exchange import allgather_packed

            result, snaps = allgather_packed(self, my_tensors, all_placeholders, target_device)
            self.last_snapshots = snaps
            return result

        # host tensors over a CPU backend: flatten, one all_gather, views
        sizes = [[tp.nbytes for tp in tps] for tps in all_placeholders]
        layouts = [_host_layout(s) for s in sizes]
        widest = max(total for _, total in layouts)
        mine = layouts[self.my_group_rank]
        send = torch.zeros(max(widest, 1), dtype=torch.uint8)
        send[: max(mine[1], 1)] = _flatten_host(my_tensors, mine[0], mine[1])
        recv = [torch.empty_like(send) for _ in range(self.world_size)]
        dist.all_gather(recv, send, group=self.group)
        result = []
        for flat, tps, (offs, _) in zip(recv, all_placeholders, layouts):
            views = _views_from_flat(flat, tps, offs)
            if target_device is not None:
                views = [v.to(target_device, non_blocking=True) for v in views]
            result.append(views)
        return result

    def all_gather_int(self, value: int) -> List[int]:
        """All-gather one int64 per rank with a plain tensor collective (no pickling): used to agree on cache keys."""
        dev = torch.device("cuda", torch.cuda.current_device()) if self.backend != "gloo" and torch.cuda.is_available() else torch.device("cpu")
        mine = torch.tensor([value], dtype=torch.int64, device=dev)
        out = torch.empty(self.world_size, dtype=torch.int64, device=dev)
        dist.all_gather_into_tensor(out, mine, group=self.group)
        return out.tolist()

    def _gather_placeholders(self, my_tensors: List[torch.Tensor]) -> List[List[TensorPlaceholder]]:
        """Shapes / dtypes of every member's tensor list.  The pickled exchange (reference ``:356-358``) is repeated only
        when some member's structure changed: every call all-gathers one 64-bit fingerprint per rank, and the vector
        of fingerprints -- identical on all members -- is the cache key."""
        import hashlib

        sig = repr([(tuple(t.shape), str(t.dtype), t.device.type, tuple(t.stride())) for t in my_tensors])
        fingerprint = int.from_bytes(hashlib.blake2b(sig.encode(), digest_size=7).digest(), "little")
        key = tuple(self.all_gather_int(fingerprint))
        cache = self.__dict__.setdefault("_placeholder_cache", {})
        if key not in cache:
            if len(cache) > 16:
                cache.clear()
            cache[key] = self.all_gather_object([TensorPlaceholder(t) for t in my_tensors])
        return cache[key]

    def isend_state_dict(self, state_dict: TensorAwareStateDict, dst: int) -> Dict[str, float]:
        """Send ``state_dict`` to global rank ``dst``: the hollow skeleton as an object, the payload as ONE
        packed message."""
        tensors = state_dict.pop_tensors()
        log = {"data_sent": sum(t.nbytes for t in tensors)}
        placeholders = [TensorPlaceholder(t) for t in tensors]
        self.send_object((state_dict, placeholders), dst)
        if log["data_sent"]:
            if self._payload_on_gpu():
                from ...b200.exchange import send_packed

                send_packed(self, tensors, dst)
            else:
                offs, total = _host_layout([tp.nbytes for tp in placeholders])
                dist.send(_flatten_host([t.cpu() for t in tensors], offs, total), dst, group=self.group)
        state_dict.insert_tensors(tensors)
        return log

    def irecv_state_dict(self, src: int):
        """Receive what ``isend_state_dict`` sent from global rank ``src``; tensors end up on the devices the
        hollow skeleton remembers."""
        hollow, placeholders = self.recv_object(src)
        hollow.init_tensors()
        dests = list(hollow.tensors)
        if self._payload_on_gpu():
            # the skeleton remembers the *sender's* device index; when sender and receiver use different local GPUs
            # (cliques inside one node) the payload must land on this rank's device, not the sender's
            here = torch.device("cuda", torch.cuda.current_device())
            moved = [torch.empty_like(d, device=here) if d.is_cuda and d.device != here else d for d in dests]
            if any(m is not d for m, d in zip(moved, dests)):
                hollow.pop_tensors()
                hollow.insert_tensors(moved)
                dests = moved
        nbytes = sum(t.nbytes for t in dests)
        if nbytes:
            if self._payload_on_gpu():
                from ...b200.exchange import recv_packed

                recv_packed(self, dests, src)
            else:
                offs, total = _host_layout([tp.nbytes for tp in placeholders])
                flat = torch.empty(max(total, 1), dtype=torch.uint8)
                dist.recv(flat, src, group=self.group)
                for dst_t, view in zip(dests, _views_from_flat(flat, placeholders, offs)):
                    dst_t.copy_(view)
        return hollow, {"data_recv": nbytes}

    def _payload_on_gpu(self) -> bool:
        """Point-to-point payloads travel through GPU memory unless the backend is CPU-only."""
        return torch.device("cuda") in [torch.device(d.type) for d in self.supported_devices] and torch.cuda.is_available()

    def _p2p_device(self) -> torch.device:
        """Where ``dist.send`` / ``dist.recv`` take their tensors: gloo reduces and gathers CUDA tensors but sends and
        receives host memory only."""
        if self._payload_on_gpu() and self.backend != dist.Backend.GLOO:
            return torch.device("cuda", torch.cuda.current_device())
        return torch.device("cpu")

    def send_tensor(self, tensor: torch.Tensor, dst: int) -> None:
        """``dist.send`` of ``tensor`` to global rank ``dst``, copied to the device the backend sends from if it is not
        there (the matching receive is :meth:`recv_tensor`)."""
        dev = self._p2p_device()
        dist.send(tensor if tensor.device.type == dev.type else tensor.to(dev), dst, group=self.group)

    def recv_tensor(self, tensor: torch.Tensor, src: int) -> None:
        """``dist.recv`` from global rank ``src`` into ``tensor`` (CUDA or host; contiguous), through a buffer on the
        device the backend receives on if ``tensor`` is elsewhere."""
        dev = self._p2p_device()
        if tensor.device.type == dev.type:
            dist.recv(tensor, src, group=self.group)
            return
        bounce = torch.empty(tensor.shape, dtype=tensor.dtype, device=dev)
        dist.recv(bounce, src, group=self.group)
        tensor.copy_(bounce)

    def execute_plan(
        self, exchange_plan: ExchangePlan, my_data: Dict[str, TensorAwareStateDict]
    ) -> Tuple[Dict[str, TensorAwareStateDict], Dict[str, float]]:
        """Carry out ``exchange_plan`` in order; returns ``{id: state_dict}`` of what this rank received
        (transfers to oneself are resolved locally)."""
        missing = exchange_plan.required_ids().difference(my_data.keys())
        assert not missing, f"Not all required data provided! Missing ids: {missing}"
        me = self.get_global_rank()
        sent_bytes = recv_bytes = 0
        received = {}
        for entry in exchange_plan.entries:
            if entry.sender == me == entry.receiver:
                received[entry.id_] = my_data[entry.id_]
            elif entry.sender == me:
                sent_bytes += self.isend_state_dict(my_data[entry.id_], entry.receiver)["data_sent"]
            elif entry.receiver == me:
                received[entry.id_], log = self.irecv_state_dict(entry.sender)
                recv_bytes += log["data_recv"]
        debug_msg(f"{sent_bytes=}")
        debug_msg(f"{recv_bytes=}")
        return received


ProcessGroupLike = Union[GroupWrapper, dist.ProcessGroup]
