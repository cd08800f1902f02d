"""NVLink peer-to-peer transport for ``PipelineCommunication`` (csrc/p2p.cu).

Host side of the mailbox rings: allocation + CUDA-IPC exchange of the mailboxes with the previous / next stage (through
the default process group's key-value store -- no collective, no extra communicator), and enqueueing the send / recv
kernels on two dedicated streams so that transfers overlap the 1F1B compute:

    send:  copy stream waits for the producing pass (event), then [wait ack] -> NVLink write -> flag
    recv:  copy stream spins on the flag, copies the slot into freshly allocated tensors, acks; the compute stream
           waits for that event only

The one-off meta handshake (pipeline.py:289-376) still runs over torch.distributed, exactly as the reference's.
"""
from __future__ import annotations

import ctypes as C
import weakref

import torch
import torch.distributed as dist

from .. import lib as L
from .pipeline import DistTransport

NSLOTS = 4
# how many links this process has created with each peer: both ends of a boundary create their n-th link at the same
# logical time (initial build, then once per reconfiguration), so (pair, n) is a collision-free rendezvous key
_LINK_SEQ: dict[tuple[int, int], int] = {}


def _align(n: int, a: int = 256) -> int:
    return (n + a - 1) // a * a


class _Link:
    """Mailbox pair with one neighbour: ``mine`` (peer writes payloads / flags / acks here) and ``peer``."""

    def __init__(self, my_rank: int, peer_rank: int, slot_bytes: int, tag: str):
        self.slot_bytes = slot_bytes
        self.mine = C.c_void_p()
        handle = (C.c_char * 64)()
        L.call("oob_p2p_alloc", NSLOTS * slot_bytes, C.byref(self.mine), handle)
        store = dist.distributed_c10d._get_default_store()
        store.set(f"oob_p2p/{tag}/{my_rank}->{peer_rank}", bytes(handle))
        peer_handle = store.get(f"oob_p2p/{tag}/{peer_rank}->{my_rank}")   # blocks until the peer has published
        self.peer = C.c_void_p()
        L.call("oob_p2p_open", C.c_char_p(bytes(peer_handle)), C.byref(self.peer))
        self.send_seq = 0
        self.recv_seq = 0

    def close(self):
        if self.peer:
            L.load().oob_p2p_close(self.peer)
            self.peer = C.c_void_p()
        if self.mine:
            L.load().oob_p2p_free(self.mine)
            self.mine = C.c_void_p()


class NvlinkRingTransport(DistTransport):
    def __init__(self, comm):
        super().__init__(comm)
        self.send_stream = torch.cuda.Stream()
        self.recv_stream = torch.cuda.Stream()
        self.links: dict[int, _Link] = {}
        self.last_send_event: torch.cuda.Event | None = None
        self._finalizer = weakref.finalize(self, NvlinkRingTransport._cleanup, self.links)

    @staticmethod
    def _cleanup(links):
        for link in links.values():
            try:
                link.close()
            except Exception:  # noqa: BLE001
                pass

    # the payload size of a link is fixed by the first tuple that crosses it (static shapes)
    def _link(self, peer_rank: int, tensors) -> _Link:
        if peer_rank not in self.links:
            slot = sum(_align(t.numel() * t.element_size()) for t in tensors)
            me = dist.get_rank()
            pair = (min(me, peer_rank), max(me, peer_rank))
            seq = _LINK_SEQ.get(pair, 0)
            _LINK_SEQ[pair] = seq + 1
            self.links[peer_rank] = _Link(me, peer_rank, self._slot_bytes(tensors, slot), f"{pair[0]}-{pair[1]}/{seq}")
        return self.links[peer_rank]

    def _slot_bytes(self, tensors, computed: int) -> int:
        # activations: (hidden f32, labels i64); gradients: (hidden-grad f32).  Allocate for hidden + labels of the
        # same leading shape so that either direction fits whichever message creates the link first.
        hidden = max((t for t in tensors if t.is_floating_point()), key=lambda t: t.numel(), default=None)
        extra = 0
        if hidden is not None and hidden.dim() == 3:
            extra = _align(hidden.shape[0] * hidden.shape[1] * 8)
        base = _align(hidden.numel() * hidden.element_size()) if hidden is not None else 0
        return max(computed, base + extra)

    def reserve_link(self, peer_rank: int, like) -> None:
        """Create the link with ``peer_rank`` now, sized for tuples shaped like ``like`` (may be meta tensors), unless
        it exists.  An evaluation pass that runs before the first training step sizes the link for the training
        tuples it sends in slices of, so that they still fit afterwards."""
        self._link(peer_rank, like)

    def send_tuple(self, tensors, dest_rank: int, kind: str):
        tensors = [t.detach().contiguous() for t in tensors]
        link = self._link(dest_rank, tensors)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream())
        self.send_stream.wait_event(ev)
        link.send_seq += 1
        off = 0
        s = C.c_void_p(self.send_stream.cuda_stream)
        for i, t in enumerate(tensors):
            nbytes = t.numel() * t.element_size()
            t.record_stream(self.send_stream)
            L.call("oob_p2p_send", C.c_void_p(t.data_ptr()), nbytes, link.mine, link.peer, NSLOTS, link.slot_bytes, off,
                   link.send_seq, int(i == 0), int(i == len(tensors) - 1), s)
            off += _align(nbytes)
        done = torch.cuda.Event()
        done.record(self.send_stream)
        self.last_send_event = done

    def _ring_recv(self, dsts, src_rank: int):
        link = self._link(src_rank, dsts)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream())
        self.recv_stream.wait_event(ev)          # destination buffers are free once prior compute has run
        link.recv_seq += 1
        off = 0
        s = C.c_void_p(self.recv_stream.cuda_stream)
        for i, t in enumerate(dsts):
            nbytes = t.numel() * t.element_size()
            t.record_stream(self.recv_stream)
            L.call("oob_p2p_recv", C.c_void_p(t.data_ptr()), nbytes, link.mine, link.peer, NSLOTS, link.slot_bytes, off,
                   link.recv_seq, int(i == 0), int(i == len(dsts) - 1), s)
            off += _align(nbytes)
        done = torch.cuda.Event()
        done.record(self.recv_stream)
        torch.cuda.current_stream().wait_event(done)

    def recv_activation_tuple(self, recv_buf: tuple, src_rank: int) -> tuple:
        fresh = [torch.empty_like(b, requires_grad=False) for b in recv_buf]   # received straight into new tensors
        self._ring_recv(fresh, src_rank)
        for t, b in zip(fresh, recv_buf):
            t.requires_grad = b.requires_grad
        return tuple(fresh)

    def recv_gradient_tuple(self, recv_buf: tuple, src_rank: int) -> None:
        self._ring_recv(list(recv_buf), src_rank)

    def before_compute(self) -> None:
        # a forward pass may overwrite a layer output buffer that an earlier SendActivation is still reading
        if self.last_send_event is not None:
            torch.cuda.current_stream().wait_event(self.last_send_event)

    def abort(self):
        """Listener thread: release every kernel of this rank that waits on a neighbour (a host store per mailbox)."""
        self._abort = True
        for link in list(self.links.values()):
            if link.mine:
                L.load().oob_p2p_abort(link.mine, None)

    def aborted(self) -> bool:
        """Host-side read of the mailboxes' control words: did any wait of this transport really give up (abort request
        honoured, or watchdog)?  Call it after the device has drained.  A bare abort request with no kernel waiting is
        not a fault: the data of the step is complete."""
        st = C.c_int(0)
        for link in list(self.links.values()):
            if link.mine and L.load().oob_p2p_status(link.mine, C.byref(st)) == 0 and st.value != 0:
                return True
        return False
