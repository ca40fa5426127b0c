"""Multi-GPU data parallelism for the forward rendering path (SURVEY.md §8e).

Every render (voxel, pose) is independent -- the forward graph has no cross-sample op -- so the path shards over
the batch axis with NO data-path collective: rank g renders items [lo, hi) of the batch with its own replica of
the weights.  The only collective is the all-gather of the output image batch the north_star asks for (plus a
one-off broadcast of the weights / the turntable voxel at start-up).  One process per GPU, torch.distributed
(NCCL on GPUs; the same code runs on gloo/CPU tensors for the host-logic tests).
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import numpy as np
import torch
import torch.distributed as dist


def shard_bounds(n_items: int, world: int, rank: int) -> Tuple[int, int]:
    """Contiguous slice of `n_items` owned by `rank`; the first n_items % world ranks get one extra item."""
    if not (0 <= rank < world):
        raise ValueError("rank out of range")
    base, extra = divmod(n_items, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def all_gather_images(local: torch.Tensor, n_total: Optional[int] = None, group=None) -> torch.Tensor:
    """[b_local,H,W,C] on every rank -> [n_total,H,W,C] on every rank (rank-major order == batch order for
    shard_bounds).  Ragged shards are padded to the largest shard for the collective and trimmed afterwards."""
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return local
    world = dist.get_world_size(group)
    if n_total is None:
        cnt = torch.tensor([local.shape[0]], device=local.device, dtype=torch.int64)
        dist.all_reduce(cnt, group=group)
        n_total = int(cnt.item())
    sizes = [shard_bounds(n_total, world, r) for r in range(world)]
    bmax = max(hi - lo for lo, hi in sizes)
    if all(hi - lo == bmax for lo, hi in sizes):
        out = torch.empty((world * bmax,) + tuple(local.shape[1:]), device=local.device, dtype=local.dtype)
        dist.all_gather_into_tensor(out, local.contiguous(), group=group)
        return out
    pad = torch.zeros((bmax,) + tuple(local.shape[1:]), device=local.device, dtype=local.dtype)
    pad[: local.shape[0]] = local
    buf = torch.empty((world * bmax,) + tuple(local.shape[1:]), device=local.device, dtype=local.dtype)
    dist.all_gather_into_tensor(buf, pad, group=group)
    parts = [buf[r * bmax: r * bmax + (hi - lo)] for r, (lo, hi) in enumerate(sizes)]
    return torch.cat(parts, dim=0)


class PeerImageGather:
    """All-gather of the per-rank image shards WITHOUT SM time: every rank owns TWO full [world*b, ...] buffers (step parity),
    exported to its peers over CUDA IPC at start-up; each step a rank writes its shard into every peer's buffer of that
    parity with plain device-to-device copies (copy engines over NVLink / NVSwitch) on a side stream.

    An alternative to ncclAllGather that leaves all SMs to the persistent convolution kernels of the next step (NCCL's
    kernels hold a few SMs while they run); `ShardedRenderEngine(gather="peer")` / `bench.py --gather peer`.

    Write-after-read safety across processes: a rank may only overwrite a peer's parity-p buffer with step i+2 after that
    peer has finished consuming step i from it.  Every rank therefore (1) records `consumed` once it is done with the
    buffer returned by the previous same-parity gather (`release()`), and (2) runs a one-element NCCL all-reduce on the side
    stream, AFTER waiting for that event and BEFORE its copies: the all-reduce completes only when every rank has passed
    its own `consumed` wait.  Single node only (IPC); construction raises if peer access or IPC is unavailable and the
    caller falls back to `all_gather_images` (NCCL)."""

    def __init__(self, shard_shape, dtype=torch.float32, device=None, group=None):
        if not dist.is_initialized():
            raise RuntimeError("PeerImageGather needs an initialised process group")
        from torch.multiprocessing.reductions import reduce_tensor
        self.group = group
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self.b = int(shard_shape[0])
        shape = (self.world * self.b,) + tuple(shard_shape[1:])
        self.full = [torch.empty(shape, device=self.device, dtype=dtype) for _ in range(2)]
        self.peers = []                                          # peers[parity][rank] aliases that rank's buffer
        for par in range(2):
            handles = [None] * self.world
            dist.all_gather_object(handles, reduce_tensor(self.full[par]), group=group)
            views = []
            for r, (rebuild, rargs) in enumerate(handles):
                if r == self.rank:
                    views.append(self.full[par])
                    continue
                t = rebuild(*rargs)                              # aliases rank r's buffer (cudaIpcOpenMemHandle)
                if not torch.cuda.can_device_access_peer(self.device.index, t.device.index):
                    raise RuntimeError(f"no peer access {self.device} -> {t.device}")
                views.append(t)
            self.peers.append(views)
        self.stream = torch.cuda.Stream(device=self.device)
        # one copy stream per destination: a single cudaMemcpyPeer stream moves ~115 GB/s on this fabric (one copy engine), the
        # world-1 outgoing copies run concurrently on separate engines
        self.copy_streams = [torch.cuda.Stream(device=self.device) for _ in range(self.world)]
        self.done = torch.cuda.Event()
        self.done.record(torch.cuda.current_stream(self.device))
        self.consumed = [torch.cuda.Event(), torch.cuda.Event()]
        for e in self.consumed:
            e.record(torch.cuda.current_stream(self.device))
        self._flag = torch.zeros(1, device=self.device)
        self.steps = 0

    def gather_async(self, local: torch.Tensor, ready: Optional[torch.cuda.Event] = None) -> torch.cuda.Event:
        """Queue the copies of `local` ([b, ...], this rank's shard) into every rank's buffer of this step's parity on the
        side stream, after `ready` (default: everything queued so far on the current stream).  Returns the event that marks
        this rank's outgoing copies complete; incoming shards are complete once every rank's event has fired (`fence()`).
        The gathered tensor of this step is `self.full[parity]` (`self.last`)."""
        if ready is None:
            ready = torch.cuda.Event()
            ready.record(torch.cuda.current_stream(self.device))
        par = self.steps % 2
        self.steps += 1
        lo = self.rank * self.b
        with torch.cuda.stream(self.stream):
            self.stream.wait_event(ready)
            self.stream.wait_event(self.consumed[par])           # this rank is done with the step-(i-2) contents ...
            dist.all_reduce(self._flag, group=self.group)        # ... and so is every other rank (see class docstring)
            go = torch.cuda.Event()
            go.record(self.stream)
        for k in range(self.world):                              # own copy first, then peers rank+1, rank+2, ...: no hot spot
            cs = self.copy_streams[k]
            with torch.cuda.stream(cs):
                cs.wait_event(go)
                self.peers[par][(self.rank + k) % self.world][lo:lo + self.b].copy_(local, non_blocking=True)
                e = torch.cuda.Event()
                e.record(cs)
            self.stream.wait_event(e)
        with torch.cuda.stream(self.stream):
            self.done = torch.cuda.Event()
            self.done.record(self.stream)
        self.last = self.full[par]
        return self.done

    def release(self, stream: Optional[torch.cuda.Stream] = None):
        """The consumer has finished (stream-ordered on `stream`, default the current one) with the buffer of the most recent
        gather: peers may overwrite it two steps from now."""
        par = (self.steps - 1) % 2
        self.consumed[par] = torch.cuda.Event()
        self.consumed[par].record(stream if stream is not None else torch.cuda.current_stream(self.device))

    def fence(self):
        """Block until every rank's outgoing copies have landed (so `self.last` is complete everywhere)."""
        self.done.synchronize()
        dist.barrier(group=self.group)

    def gather(self, local: torch.Tensor) -> torch.Tensor:
        self.gather_async(local)
        self.fence()
        self.release()
        return self.last

    def close(self):
        """Drop the peer mappings before the owners free their buffers."""
        self.fence()
        self.peers = [[self.full[0]], [self.full[1]]]
        dist.barrier(group=self.group)


class ShardedRenderEngine:
    """Batch-sharded rendering over the ranks of a process group (SURVEY §8e): every rank renders ITS `engine.B` items
    with its own weight replica (no data-path collective); the only exchange is the all-gather of the output image batch,
    issued on a side stream so that it overlaps the next step's convolutions.

        sh = ShardedRenderEngine(engine, gather="nccl")      # "nccl" | "peer" (copy engines over CUDA IPC) | "none"
        sh.step()                    # inputs already resident: graph replay + async gather
        sh.submit(vox, poses)        # or the pipelined host path: H2D -> graph -> gather (D2H of the local shard overlaps)
        full = sh.wait()             # [world*B,512,512,3] of the LAST step, complete on this rank's current stream

    With world == 1 (or no process group) it degenerates to the engine itself."""

    def __init__(self, engine, gather: str = "nccl_sync", group=None):
        """gather: "nccl_sync" (default) = ncclAllGather on the COMPUTE stream right after the step, straight from the engine's
        output buffer; "nccl" = the same collective on a side stream, overlapped with the next step; "peer" = copy-engine P2P
        writes (PeerImageGather); "none".  Overlapping the gather with the next step cannot hide much because the persistent
        convolution kernels occupy every SM (NCCL's CTAs only get SMs at kernel boundaries).  The stream-ordered form needs
        no staging copy and no second gathered buffer in flight."""
        if gather not in ("nccl", "nccl_sync", "peer", "none"):
            raise ValueError("gather must be nccl_sync | nccl | peer | none")
        self.engine, self.group = engine, group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.kind = gather if self.world > 1 else "none"
        self.dev = engine.device
        self.timing = None                           # set to [] to record per-step phase timestamps (bench.py --phases)
        outs = list(engine.outputs) if not isinstance(engine.out, torch.Tensor) else [engine.out]   # Texture engine: 2 images
        self._multi = not isinstance(engine.out, torch.Tensor)
        self.peer = None
        self.kind_note = {"nccl": "NCCL all-gather on a side stream, overlapped with the next step",
                          "nccl_sync": "NCCL all-gather on the compute stream between steps",
                          "none": "no gather (per-rank outputs only)"}.get(self.kind, "")
        if self.kind == "peer" and len(outs) != 1:
            self.kind, self.kind_note = "nccl", "NCCL all-gather (peer gather handles one output tensor)"
        if self.kind == "peer":
            ok = 1
            try:
                self.peer = PeerImageGather(tuple(outs[0].shape), outs[0].dtype, self.dev, group)
            except Exception as e:  # noqa: BLE001
                import sys
                print(f"[ShardedRenderEngine] rank {self.rank}: peer gather unavailable ({type(e).__name__}: {e}); using NCCL",
                      file=sys.stderr)
                ok = 0
            flag = torch.tensor([ok], device=self.dev)
            dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=group)          # all ranks must agree
            if int(flag.item()) == 0:
                self.peer, self.kind, self.kind_note = None, "nccl", "NCCL all-gather (peer gather unavailable)"
            else:
                self.kind_note = "copy-engine P2P writes over NVLink (CUDA IPC)"
        if self.kind in ("nccl", "nccl_sync"):
            self.comm = torch.cuda.Stream(device=self.dev) if self.kind == "nccl" else None     # side stream of the overlapped form
            self.gathered = [torch.empty((self.world * o.shape[0],) + tuple(o.shape[1:]), device=self.dev, dtype=o.dtype)
                             for o in outs]
        if self.kind in ("nccl", "peer"):
            self.src = [torch.empty_like(o) for o in outs]       # the graph overwrites the engine's outputs every step
            self.ev_ready, self.ev_done = torch.cuda.Event(), torch.cuda.Event()
            self.ev_done.record(torch.cuda.current_stream(self.dev))

    def _engine_outs(self):
        return list(self.engine.out) if self._multi else [self.engine.out]

    def verify_peer_against_nccl(self) -> bool:
        """One-off check of the peer path against ncclAllGather on a recognisable pattern (all ranks call it)."""
        if self.peer is None:
            return True
        b = self.src[0].shape[0]
        pat = torch.full_like(self.src[0], float(self.rank + 1))
        pat[:, 0, 0, 0] = torch.arange(b, device=self.dev, dtype=pat.dtype)
        got = self.peer.gather(pat).clone()
        want = torch.empty((self.world * b,) + tuple(pat.shape[1:]), device=self.dev, dtype=pat.dtype)
        dist.all_gather_into_tensor(want, pat, group=self.group)
        same = torch.tensor([int(torch.equal(got, want))], device=self.dev)
        dist.all_reduce(same, op=dist.ReduceOp.MIN, group=self.group)
        return int(same.item()) == 1

    def _gather(self):
        if self.kind == "none":
            return
        if self.kind == "nccl_sync":                 # stream-ordered between this step and the next: no copy, no overlap
            for g, o in zip(self.gathered, self._engine_outs()):
                dist.all_gather_into_tensor(g, o, group=self.group)
            return
        cur = torch.cuda.current_stream(self.dev)
        cur.wait_event(self.ev_done)                 # the previous gather has consumed self.src
        for s_, o in zip(self.src, self._engine_outs()):
            s_.copy_(o)
        self.ev_ready.record(cur)
        if self.peer is not None:
            self.peer.release(cur)                   # nothing on this rank reads the older same-parity buffer any more
            self.ev_done = self.peer.gather_async(self.src[0], self.ev_ready)
        else:
            with torch.cuda.stream(self.comm):
                self.comm.wait_event(self.ev_ready)
                for g, s_ in zip(self.gathered, self.src):
                    dist.all_gather_into_tensor(g, s_, group=self.group)
                self.ev_done = torch.cuda.Event()
                self.ev_done.record(self.comm)

    def step(self):
        if self.timing is not None:                  # per-step device timestamps: [start, compute done, gather issued/done]
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            cur = torch.cuda.current_stream(self.dev)
            ev[0].record(cur)
            self.engine.step_device()
            ev[1].record(cur)
            self._gather()
            ev[2].record(cur)
            self.timing.append(ev)
            return
        self.engine.step_device()
        self._gather()

    def phase_times(self):
        """(mean compute ms, mean gather ms on the compute stream, mean step-to-step ms) of the steps recorded since `timing = []`;
        call after a synchronize."""
        t = self.timing or []
        if not t:
            return None
        comp = sum(e[0].elapsed_time(e[1]) for e in t) / len(t)
        gath = sum(e[1].elapsed_time(e[2]) for e in t) / len(t)
        period = (t[0][0].elapsed_time(t[-1][0]) / (len(t) - 1)) if len(t) > 1 else comp + gath
        return comp, gath, period

    def submit(self, *host_inputs) -> int:
        t = self.engine.submit(*host_inputs)
        self._gather()
        return t

    def wait(self):
        """Make the current stream wait for the last step's gather; returns the gathered batch (a tuple for the two-output
        Texture engine; this rank's own images when there is no gather)."""
        if self.kind == "none":
            return self.engine.out
        if self.kind == "nccl_sync":
            return tuple(self.gathered) if self._multi else self.gathered[0]
        torch.cuda.current_stream(self.dev).wait_event(self.ev_done)
        if self.peer is not None:
            return self.peer.last
        return tuple(self.gathered) if self._multi else self.gathered[0]

    def close(self):
        if self.peer is not None:
            self.peer.close()
            self.peer = None


def all_reduce_gradients(grads: Dict[str, torch.Tensor], average: bool = True, bucket_bytes: int = 256 << 20, group=None):
    """Data-parallel training: sum (or average) every gradient of `grads` over the ranks, in place.  The tensors are packed,
    in name order (identical on every rank), into flat fp32 buckets of <= bucket_bytes so that the 166 variables of the Shader
    network cost a handful of all-reduces sized for NVSwitch bandwidth rather than 166 latency-bound ones (the 1024 x 1024
    3 x 3 filters are 37.7 MB each and travel alone-ish; biases and slopes share a bucket).  Backend-agnostic (NCCL on GPUs,
    gloo in the CPU tests)."""
    if not (dist.is_available() and dist.is_initialized()):
        return grads
    world = dist.get_world_size(group)
    if world == 1:
        return grads
    names = sorted(grads)
    i = 0
    while i < len(names):
        j, size = i, 0
        while j < len(names) and (j == i or size + grads[names[j]].numel() * 4 <= bucket_bytes):
            size += grads[names[j]].numel() * 4
            j += 1
        chunk = [grads[n] for n in names[i:j]]
        if len(chunk) == 1 and chunk[0].is_contiguous() and chunk[0].dtype == torch.float32:
            flat = chunk[0].view(-1)                       # big filters: reduce in place, no staging copy
            dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
            if average:
                flat.mul_(1.0 / world)
        else:
            flat = torch.cat([t.reshape(-1).float() for t in chunk])
            dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
            if average:
                flat.mul_(1.0 / world)
            off = 0
            for t in chunk:
                t.copy_(flat[off:off + t.numel()].view(t.shape))
                off += t.numel()
        i = j
    return grads


def broadcast_weight_dict(weights: Optional[Dict[str, np.ndarray]], src: int = 0, device="cpu", group=None):
    """Replicate a weight dict from `src` to every rank (names first, then one flat fp32 buffer)."""
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return weights
    meta = [[(k, tuple(np.asarray(v).shape)) for k, v in sorted(weights.items())]] if dist.get_rank(group) == src else [None]
    dist.broadcast_object_list(meta, src=src, group=group)
    names = meta[0]
    total = sum(int(np.prod(s)) for _, s in names)
    flat = torch.empty(total, dtype=torch.float32, device=device)
    if dist.get_rank(group) == src:
        flat.copy_(torch.cat([torch.as_tensor(np.asarray(weights[k], np.float32)).reshape(-1) for k, _ in names]))
    dist.broadcast(flat, src=src, group=group)
    out, off = {}, 0
    flat_cpu = flat.cpu().numpy()
    for k, s in names:
        n = int(np.prod(s))
        out[k] = flat_cpu[off:off + n].reshape(s)
        off += n
    return out


def turntable_poses(n_frames: int = 360, elevation: float = 60.0, radius: float = 3.3, step_deg: Optional[float] = None):
    """Poses of the demo's azimuth sweep (RenderNet_demo.py:133: 0..355 step 5; BASELINE config 5: 0..359 step 1)."""
    step = step_deg if step_deg is not None else 360.0 / n_frames
    az = np.arange(n_frames, dtype=np.float64) * step
    return np.stack([az * math.pi / 180.0, np.full(n_frames, (90 - elevation) * math.pi / 180),
                     np.full(n_frames, 3.3 / radius)], axis=1).astype(np.float32)
