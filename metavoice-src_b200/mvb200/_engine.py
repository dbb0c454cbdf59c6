"""Host plumbing shared by every wrapper of a libmvb200 engine handle: the weight-arena format, the handle's lifetime,
the stream its calls go on and how a batch is split to fit a batch workspace."""
from __future__ import annotations

import ctypes as C
from typing import List, Sequence, Tuple

import torch

from . import _lib

ALIGN = 256  # byte alignment of every tensor inside a weight arena (TMA needs >= 128; check_offsets in C needs >= 16)


def align_up(n: int) -> int:
    return (n + ALIGN - 1) // ALIGN * ALIGN


def pack_arena_bytes(blobs: Sequence[torch.Tensor]) -> Tuple[torch.Tensor, List[int]]:
    """Tensors of any dtype -> (uint8 arena on the CPU, byte offsets): each tensor's raw bytes at the next 256-byte
    boundary, in order, with zero padding.  Each engine chooses its tensors' dtypes before packing."""
    flat = [b.detach().contiguous().reshape(-1).view(torch.uint8) for b in blobs]
    offsets: List[int] = []
    total = 0
    for b in flat:
        offsets.append(total)
        total = align_up(total + b.numel())
    arena = torch.zeros(total, dtype=torch.uint8)
    for b, o in zip(flat, offsets):
        arena[o:o + b.numel()] = b
    return arena, offsets


def split_runs(sizes: Sequence[int], max_items: int, max_total: int) -> List[range]:
    """Consecutive runs of indices into ``sizes`` with at most ``max_items`` items and a total size of at most
    ``max_total`` each.  An item larger than ``max_total`` forms a run of its own, which the library call rejects."""
    runs, s0, tot = [], 0, 0
    for i, n in enumerate(sizes):
        if i > s0 and (i - s0 == max_items or tot + n > max_total):
            runs.append(range(s0, i))
            s0, tot = i, 0
        tot += n
    if s0 < len(sizes):
        runs.append(range(s0, len(sizes)))
    return runs


def current_stream(device: torch.device) -> C.c_void_p:
    """The current PyTorch stream of ``device``, as the ``stream`` argument of a libmvb200 call."""
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


class Engine:
    """One libmvb200 engine handle and the device memory it was created over: the weight arena and the workspaces."""

    _h = None  # the handle; None before _create succeeds and after close()

    def __init__(self, device, arena: torch.Tensor, offsets: Sequence[int]):
        self.device = torch.device(device)
        self._lib = _lib.load()
        self._arena = arena.to(self.device)
        self._offsets = list(offsets)

    def _create(self, create, destroy, cfg, *workspace_bytes) -> None:
        """One zeroed device workspace of ``size(cfg)`` bytes per function in ``workspace_bytes`` (a size of 0 means the
        library does not support ``cfg``), kept in ``self._ws``; then ``create(cfg, arena, arena bytes, offsets,
        *workspaces, &handle)`` on the engine's device.  close() frees the handle with ``destroy``; after it, _create may
        be called again."""
        sizes = [size(C.byref(cfg)) for size in workspace_bytes]
        if 0 in sizes:
            _lib.check(_lib.MVB_ERR_UNSUPPORTED)
        self._ws = None  # a re-created engine's old workspaces go before the new ones are allocated
        self._ws = [torch.zeros(n, dtype=torch.uint8, device=self.device) for n in sizes]
        offs = (C.c_uint64 * len(self._offsets))(*self._offsets)
        h = C.c_void_p()
        torch.cuda.synchronize(self.device)  # the zero fills run on the current stream; create may use its own
        with torch.cuda.device(self.device):
            rc = create(C.byref(cfg), self._arena.data_ptr(), self._arena.numel(), offs, *(w.data_ptr() for w in self._ws),
                        C.byref(h))
        _lib.check(rc)
        self._h, self._destroy = h, destroy

    def _batch_workspace_of(self, nbytes: int, zeroed: bool = True) -> torch.Tensor:
        """A device batch workspace of ``nbytes``; a size of 0 means the library rejected the batch shape."""
        if nbytes == 0:
            _lib.check(_lib.MVB_ERR_ARG)
        return (torch.zeros if zeroed else torch.empty)(nbytes, dtype=torch.uint8, device=self.device)

    def _st(self) -> C.c_void_p:
        return current_stream(self.device)

    def close(self):
        if self._h is not None:
            h, self._h = self._h, None
            self._destroy(h)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
