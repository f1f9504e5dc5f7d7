"""Multi-GPU: independent clips shard data-parallel, one process per GPU (SURVEY.md §8e: "replicas only").

Frame i of a clip consumes stylized frame i-1 (fast_artistic_video.lua:153-158,168-169), so nothing inside a clip
parallelises over time; clips share only read-only weights.  The only communication is moving inputs from the rank
that decoded them to the owning rank and collecting outputs -- torch.distributed point-to-point (NCCL over NVLink on
the GPU box, gloo in the CPU tests).  No collective sits on the data path of a frame.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch
import torch.distributed as dist


def assign_clips(num_clips: int, world_size: int) -> List[List[int]]:
    """Round-robin: clip c is owned by rank c % world_size."""
    return [[c for c in range(num_clips) if c % world_size == r] for r in range(world_size)]


def owner(clip: int, world_size: int) -> int:
    return clip % world_size


def scatter_clips(clips: Optional[List[torch.Tensor]], shapes: List[tuple], src: int = 0, device=None,
                  dtype=torch.float32) -> Dict[int, torch.Tensor]:
    """Rank `src` holds clips[c] (any tensor per clip, e.g. [T,3,H,W] frames); every rank returns {clip: tensor} for the
    clips it owns.  shapes[c] is known on all ranks (from the container headers)."""
    rank, world = dist.get_rank(), dist.get_world_size()
    mine: Dict[int, torch.Tensor] = {}
    reqs = []
    for c, shp in enumerate(shapes):
        o = owner(c, world)
        if rank == src:
            if o == src:
                mine[c] = clips[c].to(device) if device is not None else clips[c]
            else:
                t = clips[c].to(device) if device is not None else clips[c]
                reqs.append(dist.isend(t.contiguous(), dst=o, tag=c))
        elif rank == o:
            buf = torch.empty(shp, dtype=dtype, device=device)
            reqs.append(dist.irecv(buf, src=src, tag=c))
            mine[c] = buf
    for r in reqs:
        r.wait()
    return mine


def gather_clips(local: Dict[int, torch.Tensor], shapes: List[tuple], dst: int = 0, device=None,
                 dtype=torch.float32) -> Optional[List[torch.Tensor]]:
    """Inverse of scatter_clips: rank `dst` returns the list of all clips' outputs, other ranks None."""
    rank, world = dist.get_rank(), dist.get_world_size()
    out: List[Optional[torch.Tensor]] = [None] * len(shapes)
    reqs = []
    for c, shp in enumerate(shapes):
        o = owner(c, world)
        if rank == dst:
            if o == dst:
                out[c] = local[c]
            else:
                buf = torch.empty(shp, dtype=dtype, device=device)
                reqs.append(dist.irecv(buf, src=o, tag=c))
                out[c] = buf
        elif rank == o:
            reqs.append(dist.isend(local[c].contiguous(), dst=dst, tag=c))
    for r in reqs:
        r.wait()
    return out if rank == dst else None


# ---------------------------------------------------------------------------------------------------------------------
# Streaming data plane (BASELINE.json config 3: 8 independent 1080p clips across 8 GPUs, "NCCL over NVLink only to scatter
# frames and gather outputs").  Rank `src` owns every clip's inputs (decoded into pinned host memory); per chunk of
# `chunk` frames it uploads the chunk and sends it to the owning rank, owners run the recurrent frame loop on their clips
# and send the stylized chunk back.  One batch_isend_irecv per chunk step (NCCL group: no ordering deadlocks); the transfers
# of chunk k+1 (inputs) and k-1 (outputs) fly while chunk k is processed.
# ---------------------------------------------------------------------------------------------------------------------
def stream_clips(num_clips, n_frames, chunk, in_shapes, out_shape, load_chunk, process_chunk, store_chunk, src=0, device=None,
                 dtype=torch.float32, in_dtypes=None, out_dtype=None):
    """in_shapes: per-frame shapes of the input tensors of a clip, e.g. [(3,H,W), (2,H,W), (2,H,W)]; out_shape e.g. (3,H,W).
    load_chunk(clip, f0, f1) -> list of tensors [f1-f0, *shape] (rank src only; host or device; moved to `device`),
    process_chunk(clip, f0, inputs) -> tensor [f1-f0, *out_shape] on `device` (owner ranks, called in frame order),
    store_chunk(clip, f0, out) (rank src only).  Returns dict(comm_wait_s, steps, bytes_in, bytes_out) of this rank.
    in_dtypes / out_dtype: element types of the travelling tensors when they are not all `dtype` (e.g. uint8 frames as the
    files hold them, uint8 PNG scanlines back).

    On a CUDA device three streams are used: the caller's current stream runs process_chunk only; a transfer stream carries
    the uploads of load_chunk and the NCCL sends / receives (so chunk k+1 travels while chunk k is processed); a third stream
    carries store_chunk (the D2H of results).  The host is never more than two chunk steps ahead of the device."""
    import contextlib
    import time

    rank, world = dist.get_rank(), dist.get_world_size()
    in_dtypes = list(in_dtypes) if in_dtypes is not None else [dtype] * len(in_shapes)
    out_dtype = out_dtype if out_dtype is not None else dtype
    nsteps = (n_frames + chunk - 1) // chunk
    mine = [c for c in range(num_clips) if owner(c, world) == rank]
    span = lambda k: (k * chunk, min(n_frames, (k + 1) * chunk))
    inbuf = {}   # (clip, k) -> list of device tensors
    outbuf = {}  # (clip, k) -> device tensor
    stats = dict(comm_wait_s=0.0, steps=nsteps, bytes_in=0, bytes_out=0)
    use_cuda = device is not None and torch.device(device).type == "cuda"
    if use_cuda:
        main = torch.cuda.current_stream(device)
        xs, ss = torch.cuda.Stream(device), torch.cuda.Stream(device)
        xs.wait_stream(main); ss.wait_stream(main)
    done_ev, xfer_ev = {}, {}  # step -> event: chunk processed (main stream) / transfers of the step complete (transfer stream)

    def on(stream):
        return torch.cuda.stream(stream) if use_cuda else contextlib.nullcontext()

    def to_dev(t):
        return t.to(device, non_blocking=True) if device is not None else t

    def exchange(k):
        """post the transfers of step k: inputs of chunk k (src -> owners) and outputs of chunk k-2 (owners -> src)"""
        ops = []
        kk = k - 2
        with on(xs if use_cuda else None):
            if use_cuda and kk in done_ev:
                xs.wait_event(done_ev[kk])  # the outputs of chunk k-2 are sent from this stream
            if 0 <= k < nsteps:
                f0, f1 = span(k)
                for c in range(num_clips):
                    o = owner(c, world)
                    if rank == src:
                        ts = [to_dev(t) for t in load_chunk(c, f0, f1)]
                        if o == src:
                            inbuf[(c, k)] = ts
                        else:
                            for t in ts:
                                ops.append(dist.P2POp(dist.isend, t.contiguous(), o))
                                stats["bytes_in"] += t.numel() * t.element_size()
                            inbuf[(c, k)] = ts  # keep alive until the send completes
                    elif rank == o:
                        ts = [torch.empty((f1 - f0,) + tuple(s), dtype=dt, device=device) for s, dt in zip(in_shapes, in_dtypes)]
                        for t in ts:
                            ops.append(dist.P2POp(dist.irecv, t, src))
                        inbuf[(c, k)] = ts
            if 0 <= kk < nsteps:
                f0, f1 = span(kk)
                for c in range(num_clips):
                    o = owner(c, world)
                    if o == src:
                        continue
                    if rank == o:
                        t = outbuf[(c, kk)].contiguous()
                        if use_cuda:
                            t.record_stream(xs)
                        ops.append(dist.P2POp(dist.isend, t, src))
                        stats["bytes_out"] += t.numel() * t.element_size()
                    elif rank == src:
                        t = torch.empty((f1 - f0,) + tuple(out_shape), dtype=out_dtype, device=device)
                        ops.append(dist.P2POp(dist.irecv, t, o))
                        outbuf[(c, kk)] = t
            return dist.batch_isend_irecv(ops) if ops else []

    def finish(works, k):
        t0 = time.perf_counter()
        with on(xs if use_cuda else None):
            for w in works:
                w.wait()  # gloo: the host waits; NCCL: the transfer stream waits
            if use_cuda:
                xfer_ev[k] = xs.record_event()
        stats["comm_wait_s"] += time.perf_counter() - t0
        kk = k - 2
        if 0 <= kk < nsteps:
            f0, _ = span(kk)
            with on(ss if use_cuda else None):
                if use_cuda:
                    ss.wait_event(xfer_ev[k])      # outputs received from the other ranks
                    if kk in done_ev:
                        ss.wait_event(done_ev[kk])  # outputs computed here
                for c in range(num_clips):
                    if rank == src:
                        t = outbuf.pop((c, kk))
                        if use_cuda:
                            t.record_stream(ss)
                        store_chunk(c, f0, t)
                    elif owner(c, world) == rank:
                        outbuf.pop((c, kk), None)
        if rank == src and 0 <= k < nsteps:  # remote clips' staging buffers of step k are on the wire no longer
            for c in range(num_clips):
                if owner(c, world) != src:
                    inbuf.pop((c, k), None)

    pending = exchange(0)
    finish(pending, 0)
    for k in range(nsteps + 2):
        pending = exchange(k + 1)          # in flight while chunk k is processed
        if k < nsteps:
            f0, _ = span(k)
            if use_cuda:
                main.wait_event(xfer_ev[k])
                if k - 2 in done_ev:
                    done_ev[k - 2].synchronize()  # throttle: the host stays at most two chunk steps ahead
            for c in mine:
                ts = inbuf.pop((c, k))
                if use_cuda:
                    for t in ts:
                        t.record_stream(main)
                outbuf[(c, k)] = process_chunk(c, f0, ts)
            if use_cuda:
                done_ev[k] = main.record_event()
        finish(pending, k + 1)
    if use_cuda:
        main.wait_stream(xs); main.wait_stream(ss)
    return stats


# ---------------------------------------------------------------------------------------------------------------------
# One GPU, many clips: B clips of one frame size advance in lockstep, one batched call per frame index.  Each clip keeps its
# own recurrent state (its previous stylized frame); every frame of clip b equals that clip's single-clip trajectory bit for
# bit (models_video.StyleNet batches, include/fav.h fav_run_next_image_batch).
# ---------------------------------------------------------------------------------------------------------------------
def run_clips_lockstep(net, frames: torch.Tensor, flows: torch.Tensor, certs: torch.Tensor, fills: Optional[torch.Tensor] = None,
                       flow_masks: Optional[torch.Tensor] = None, border_mode: int = 0, styles=None) -> torch.Tensor:
    """frames [B,T,3,H,W] RGB in [0,1]; flows [B,T,2,H,W] (dy,dx) and certs [B,T,H,W], entry t used for frame t >= 1 (entry 0 is
    ignored); fills / flow_masks [B,T,3,H,W] / [B,T,H,W] or None.  Frame 0 of every clip goes through run_image (batched),
    frame t >= 1 through run_next_image on the clips' frames t - 1.  styles: None, or the style of each clip in net's style bank
    (StyleNet.add_style): clip b then equals that clip run alone on the net its style came from.  Returns the stylized frames
    [B,T,3,H,W]."""
    B, T = frames.shape[:2]
    out = torch.empty_like(frames)
    pick = lambda t, i: None if t is None else t[:, i].contiguous()
    out[:, 0] = net.run_image(frames[:, 0].contiguous(), pick(fills, 0), styles=styles)
    for i in range(1, T):
        out[:, i] = net.run_next_image(frames[:, i].contiguous(), out[:, i - 1].contiguous(), flows[:, i].contiguous(),
                                       certs[:, i].contiguous(), pick(fills, i), pick(flow_masks, i), border_mode, styles=styles)
    return out
