"""Multi-GPU partitioning of a clip (SURVEY.md §8e) and the peer-memory plumbing for the motion-module exchange.

One process per GPU. A clip offers three communication-free axes and one that needs an exchange:

  * the two classifier-free-guidance branches (pipeline :385-391, :545-549): exchange eps once per step;
  * the context windows of a long clip (pipeline :492-546): overlapping frames are summed once per step;
  * the frames inside a window: everything in UNet3DConditionModel.forward is per frame EXCEPT the temporal
    attention (motion_module.py:353-390) — around each motion module the tokens are re-sharded frames <-> pixels by
    mimo_exchange (csrc/exchange.cu): peer loads over NVLink, no NCCL on the data path.

ShardPlan picks (cfg_ways, win_ways, frame_ways) with cfg_ways * win_ways * frame_ways == world: whole windows
first, then frames, the CFG pair last (it is free of communication but unbalanced: the conditional branch attends to
twice the keys, so the unconditional GPU waits for the conditional one at every step).
torch.distributed is used for bootstrap only (exchanging 64-byte IPC handles) and for the once-per-clip gathers.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from .. import lib as L


@dataclass(frozen=True)
class ShardPlan:
    world: int
    rank: int
    cfg_ways: int
    win_ways: int
    frame_ways: int

    @staticmethod
    def make(world: int, rank: int, do_cfg: bool, n_windows: int, window_frames: int,
             min_tokens: Optional[int] = None) -> "ShardPlan":
        """Windows first (communication-free, balanced), then frames (one exchange pair per motion module, balanced),
        the CFG pair last: it needs no exchange but is UNBALANCED - the conditional branch attends to twice the keys at
        every spatial attention (the unconditional GPU waits for the conditional one), so it is only used
        for what the other two axes cannot divide. min_tokens: tokens per frame at the coarsest UNet level (each frame
        group member owns min_tokens / frame_ways of them)."""
        if world < 1 or not 0 <= rank < world:
            raise ValueError(f"bad world/rank {world}/{rank}")
        best = None
        for win_ways in sorted((d for d in range(1, world + 1) if world % d == 0 and n_windows % d == 0), reverse=True):
            rest = world // win_ways
            for frame_ways in sorted((d for d in range(1, rest + 1) if rest % d == 0), reverse=True):
                cfg_ways = rest // frame_ways
                if window_frames % frame_ways or (min_tokens is not None and min_tokens % frame_ways):
                    continue
                if cfg_ways > (2 if do_cfg else 1):
                    continue
                best = (cfg_ways, win_ways, frame_ways)
                break
            if best:
                break
        if best is None:
            raise NotImplementedError(f"{world} GPUs cannot partition {n_windows} window(s) of {window_frames} frames "
                                      f"(cfg={do_cfg}): frames per window must divide evenly")
        return ShardPlan(world, rank, *best)

    # rank = (win_idx * cfg_ways + cfg_idx) * frame_ways + frame_idx : a frame group is a run of consecutive ranks
    def coords(self, rank: Optional[int] = None) -> Tuple[int, int, int]:
        r = self.rank if rank is None else rank
        return r // (self.cfg_ways * self.frame_ways), (r // self.frame_ways) % self.cfg_ways, r % self.frame_ways

    @property
    def win_idx(self) -> int:
        return self.coords()[0]

    @property
    def cfg_idx(self) -> int:
        return self.coords()[1]

    @property
    def frame_idx(self) -> int:
        return self.coords()[2]

    def frame_group(self) -> List[int]:
        base = self.rank - self.frame_idx
        return list(range(base, base + self.frame_ways))

    def branches(self, do_cfg: bool, rank: Optional[int] = None) -> Tuple[int, ...]:
        """CFG branches (0 = unconditional, 1 = conditional) a rank evaluates."""
        if not do_cfg:
            return (0,)
        return (self.coords(rank)[1],) if self.cfg_ways == 2 else (0, 1)

    def windows_of(self, n_windows: int, rank: Optional[int] = None) -> List[int]:
        w = self.coords(rank)[0]
        return [i for i in range(n_windows) if i % self.win_ways == w]

    def local_frames(self, window: Sequence[int], rank: Optional[int] = None) -> List[int]:
        """This rank's contiguous slice of a window's frame list (window order, so PE rows stay global positions)."""
        fl = len(window) // self.frame_ways
        k = self.coords(rank)[2]
        return list(window[k * fl:(k + 1) * fl])


def gather_layout(plan: ShardPlan, windows: Sequence[Sequence[int]], do_cfg: bool):
    """Where every slice of the per-step all-gather lands. Each rank contributes one [branches, 4, fl, h, w] prediction
    per window it owns (slot j = its j-th window); returns [(rank q, slot j, branches of q, frame indices)] in
    ascending window order — the order in which the reference accumulates windows (pipeline :540-542)."""
    n = len(windows)
    per_rank = len(plan.windows_of(n, 0))
    order = sorted((plan.windows_of(n, q)[j], q, j) for q in range(plan.world) for j in range(per_rank))
    return [(q, j, plan.branches(do_cfg, q), plan.local_frames(windows[wi], q)) for wi, q, j in order]


# ------------------------------------------------------------------------------------------------
# peer memory
# ------------------------------------------------------------------------------------------------
class _RawCuda:
    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3,
                                         "strides": None}


def _as_tensor(ptr: int, nbytes: int, device) -> torch.Tensor:
    return torch.as_tensor(_RawCuda(ptr, nbytes), device=device)


class PeerBuffer:
    """`nbytes` of device memory on every member of a group, each member's copy mapped into every other member."""

    def __init__(self, nbytes: int, local_ptr: int, peer_ptrs: List[int], device, owned: bool):
        self.nbytes, self.ptr, self.peer_ptrs, self.device, self._owned = nbytes, local_ptr, peer_ptrs, device, owned
        self.bytes = _as_tensor(local_ptr, nbytes, device)

    def view(self, rows: int, cols: int, dtype: torch.dtype) -> torch.Tensor:
        n = rows * cols * torch.empty((), dtype=dtype).element_size()
        if n > self.nbytes:
            raise L.MimoError(f"peer buffer of {self.nbytes} bytes is too small for [{rows}, {cols}] {dtype}")
        return self.bytes[:n].view(dtype).view(rows, cols)


def _alloc_local(nbytes: int) -> Tuple[int, bytes]:
    ptr = C.c_void_p()
    h = C.create_string_buffer(64)
    L.check(L.load().mimo_peer_alloc(int(nbytes), C.byref(ptr), h), "mimo_peer_alloc")
    return ptr.value, h.raw


def alloc_peer_buffers(sizes: Sequence[int], members: Sequence[int], rank: int, device, group=None) -> List[PeerBuffer]:
    """Collective over the WHOLE process group `group` (every rank calls it with the same `sizes`): allocates one
    shareable buffer per entry, all-gathers the IPC handles and maps the buffers of `members` (global ranks, must
    include `rank`) into this process."""
    import torch.distributed as dist
    mine = [_alloc_local(max(int(s), 256)) for s in sizes]
    handles: List[Optional[list]] = [None] * dist.get_world_size(group)
    dist.all_gather_object(handles, [h for _, h in mine], group=group)
    out = []
    for i, (ptr, _) in enumerate(mine):
        peers = []
        for m in members:
            if m == rank:
                peers.append(ptr)
            else:
                p = C.c_void_p()
                L.check(L.load().mimo_peer_open(handles[m][i], C.byref(p)), f"mimo_peer_open(rank {m})")
                peers.append(p.value)
        out.append(PeerBuffer(max(int(sizes[i]), 256), ptr, peers, device, True))
    dist.barrier(group)  # nobody proceeds (and possibly frees) before everyone has mapped everything
    return out


class Exchange:
    """One member's handle on a frame group: flags + the two source buffers (A: frames->pixels, B: pixels->frames) and
    an all-gather source (S). `pull` enqueues one mimo_exchange on the current stream."""

    def __init__(self, G: int, r: int, flags: PeerBuffer, bufs: Dict[str, PeerBuffer], device, timeout_ms: int = 0,
                 max_blocks: int = 0):
        self.G, self.r, self.flags, self.bufs, self.device = G, r, flags, bufs, device
        self.ctl = torch.tensor([1, 0], dtype=torch.int32, device=device)
        self.timeout_ms, self.max_blocks = timeout_ms, max_blocks

    @staticmethod
    def local_group(G: int, sizes: Dict[str, int], device, **kw) -> List["Exchange"]:
        """G members inside ONE process on one device (tests, and a way to exercise the protocol on a single GPU):
        the members' kernels must run concurrently (one stream each, few blocks) because they wait for each other."""
        flags = [torch.zeros(L.MAX_PEERS, dtype=torch.int32, device=device) for _ in range(G)]
        raw = {k: [torch.zeros(max(v, 256), dtype=torch.uint8, device=device) for _ in range(G)] for k, v in sizes.items()}
        out = []
        for r in range(G):
            fb = PeerBuffer(4 * L.MAX_PEERS, flags[r].data_ptr(), [f.data_ptr() for f in flags], device, False)
            bufs = {k: PeerBuffer(max(sizes[k], 256), raw[k][r].data_ptr(), [t.data_ptr() for t in raw[k]], device, False)
                    for k in sizes}
            ex = Exchange(G, r, fb, bufs, device, **kw)
            ex._keep = (flags, raw)
            out.append(ex)
        return out

    @staticmethod
    def create(members: Sequence[int], rank: int, sizes: Dict[str, int], device, group=None, **kw) -> "Exchange":
        """Collective over `group` (all ranks, also those in other frame groups, call it with the same sizes)."""
        names = sorted(sizes)
        pbs = alloc_peer_buffers([4 * L.MAX_PEERS] + [sizes[k] for k in names], members, rank, device, group)
        return Exchange(len(members), list(members).index(rank), pbs[0], dict(zip(names, pbs[1:])), device, **kw)

    def destroy(self, group=None) -> None:
        """Collective: unmap the peers' buffers, then (after everyone has unmapped) free this member's own. Nothing may
        still be queued on these buffers - in particular no captured CUDA graph may be replayed afterwards."""
        import torch.distributed as dist
        torch.cuda.synchronize(self.device)
        pbs = [self.flags] + list(self.bufs.values())
        if not all(pb._owned for pb in pbs):
            return
        dist.barrier(group)
        for pb in pbs:
            for s, ptr in enumerate(pb.peer_ptrs):
                if s != self.r:
                    L.check(L.load().mimo_peer_close(C.c_void_p(ptr)), "mimo_peer_close")
        dist.barrier(group)
        for pb in pbs:
            pb.bytes = None
            L.check(L.load().mimo_peer_free(C.c_void_p(pb.ptr)), "mimo_peer_free")
            pb._owned = False

    def pull(self, mode: int, name: str, dst: torch.Tensor, b: int, fl: int, hw: int, Cdim: int,
             residual: Optional[torch.Tensor] = None) -> torch.Tensor:
        from .. import ops
        return ops.exchange(self, mode, name, dst, b, fl, hw, Cdim, residual)
