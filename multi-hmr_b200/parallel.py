"""Image-level data parallelism over the GPUs of one box (SURVEY.md §8e).

The reference is single-GPU with no collectives (README.md:107); images are independent units of
`Model.forward`, so the batch is split into contiguous shards, every rank runs the full single-GPU engine
on its shard with replicated weights, and ONE all-gather of a compact per-rank record block (count in the
header) returns the result to every rank: `mhmr_pack_records` + `mhmr_allgather_records` behind the C-ABI on
GPUs (NCCL over NVLink), torch.distributed/gloo with the same block layout in the CPU tests.  Ordering after the
gather is rank-major = global (b, y, x) order because the shards are contiguous.
"""
from __future__ import annotations

import torch
import torch.distributed as dist

from . import _lib
from ._lib import call

# per-person record layout (fp32): [global image index, score, loc(2), transl(3), transl_pelvis(3),
# rotvec(159), expression(10), shape(nb), v3d(3V), j3d(381), j2d(254)]
FIELDS = (("img", 1), ("scores", 1), ("loc", 2), ("transl", 3), ("transl_pelvis", 3), ("rotvec", 159),
          ("expression", 10))


def shard_range(batch: int, world: int, rank: int) -> tuple[int, int]:
    """Contiguous shard [lo, hi) of `batch` images for `rank`; the first batch % world ranks get one more."""
    base, rem = divmod(batch, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def record_layout(num_betas: int, num_verts: int):
    fields = FIELDS + (("shape", num_betas), ("v3d", 3 * num_verts), ("j3d", 381), ("j2d", 254))
    offs, o = {}, 0
    for name, n in fields:
        offs[name] = (o, n)
        o += n
    return offs, o


HEADER_WORDS = 8  # int32: persons detected, persons packed, capacity, floats per record, first global image, 0, 0, 0


def pack_block_torch(t: dict, P: int, img_offset: int, capacity: int, num_betas: int, num_verts: int) -> torch.Tensor:
    """Plain-torch statement of the record block that `mhmr_pack_records` (csrc/gather.cu) writes with ONE
    kernel: [header | capacity x record] as a flat fp32 tensor (header words are int32 bit patterns).  Used by
    the CPU (gloo) tests of the host logic and as the checker of the kernel in the GPU tests."""
    offs, R = record_layout(num_betas, num_verts)
    dev = t["v3d"].device
    block = torch.zeros(HEADER_WORDS + capacity * R, device=dev, dtype=torch.float32)
    packed = min(P, capacity)
    block[:HEADER_WORDS].view(torch.int32).copy_(
        torch.tensor([P, packed, capacity, R, img_offset, 0, 0, 0], dtype=torch.int32))
    if packed > 0:
        rec = block[HEADER_WORDS:].view(capacity, R)
        src = {"img": (t["det_idx"][0, :packed].float() + img_offset)[:, None], "scores": t["det_score"][:packed, None],
               "loc": t["loc"][:packed], "transl": t["transl"][:packed], "transl_pelvis": t["transl_pelvis"][:packed],
               "rotvec": t["rotvec"][:packed].reshape(packed, -1), "expression": t["expression"][:packed],
               "shape": t["shape"][:packed], "v3d": t["v3d"][:packed].reshape(packed, -1),
               "j3d": t["j3d"][:packed].reshape(packed, -1), "j2d": t["j2d"][:packed].reshape(packed, -1)}
        for name, (o, n) in offs.items():
            rec[:packed, o:o + n] = src[name]
    return block


def split_blocks(all_blocks: torch.Tensor, world: int, capacity: int, R: int):
    """[world * block] -> (per-rank detected counts, per-rank packed counts, valid records in rank order).
    Reads the headers on the host (one small D2H copy)."""
    blocks = all_blocks.view(world, HEADER_WORDS + capacity * R)
    hdr = blocks[:, :HEADER_WORDS].contiguous().view(torch.int32).cpu()
    detected, packed = hdr[:, 0].tolist(), hdr[:, 1].tolist()
    recs = [blocks[r, HEADER_WORDS:].view(capacity, R)[:packed[r]] for r in range(world)]
    return detected, packed, torch.cat(recs, dim=0)


def unpack_records(rec: torch.Tensor, num_betas: int, num_verts: int) -> list[dict]:
    """[P, R] -> list of person dicts with the reference's keys (model.py:329-347) + 'img' (global index)."""
    offs, _ = record_layout(num_betas, num_verts)
    shapes = {"loc": (2,), "transl": (3,), "transl_pelvis": (1, 3), "rotvec": (53, 3), "expression": (10,),
              "shape": (num_betas,), "v3d": (num_verts, 3), "j3d": (127, 3), "j2d": (127, 2)}
    persons = []
    for i in range(rec.shape[0]):
        p = {"img": int(rec[i, 0].item()), "scores": rec[i, 1]}
        for name, shp in shapes.items():
            o, n = offs[name]
            p[name] = rec[i, o:o + n].reshape(shp)
        persons.append(p)
    return persons


class RecordGather:
    """The exchange step of a sharded batch: pack (one kernel) + ONE all-gather of the per-rank record blocks,
    enqueued on a side stream so that the next forward of this rank overlaps it; the person count travels in the
    block header, so nothing is read back on the host until the caller asks for the result.

    On CUDA the collective goes through the C-ABI (`mhmr_pack_records` / `mhmr_allgather_records`, its own NCCL
    communicator bootstrapped over the default process group).  Without CUDA (gloo tests of the host logic) the
    same block layout is packed with torch ops and gathered with torch.distributed.

    capacity: record slots per rank in the gathered block (default: 4 per image of the shard, at least 8).  When
    some rank detected more, a second, full-size round is run (decided from the gathered headers, identically on
    every rank), so nothing is ever truncated."""

    def __init__(self, model, rank=None, world=None, group=None, capacity=None):
        self.model, self.group = model, group
        self.rank = dist.get_rank(group) if rank is None else rank
        self.world = dist.get_world_size(group) if world is None else world
        self.nb, self.V, self.Pm = model.num_betas, model.num_verts, model.max_persons
        _, self.R = record_layout(self.nb, self.V)
        self.capacity = int(min(self.Pm, capacity if capacity is not None else max(8, 4 * model.max_batch)))
        self.cuda = torch.cuda.is_available() and getattr(model, "device", torch.device("cpu")).type == "cuda"
        self._pending = None
        self._comm = None
        if self.cuda:
            self._init_cuda()

    # ---- CUDA path -------------------------------------------------------------------------------
    def _init_cuda(self):
        dev = self.model.device
        uid = torch.zeros(128, dtype=torch.uint8)
        if self.rank == 0:
            call("mhmr_nccl_unique_id", uid)
        uid = uid.to(dev)
        dist.broadcast(uid, src=0, group=self.group)
        comm = torch.zeros(1, dtype=torch.int64)
        with torch.cuda.device(dev):
            call("mhmr_comm_create", uid.cpu(), self.world, self.rank, comm)
        self._comm = comm.item()
        self.stream = torch.cuda.Stream(device=dev)
        self._bufs = {}

    def _buffers(self, capacity):
        if capacity not in self._bufs:
            n = HEADER_WORDS + capacity * self.R
            dev = self.model.device
            self._bufs[capacity] = (torch.empty(n, device=dev), torch.empty(self.world * n, device=dev))
        return self._bufs[capacity]

    def _enqueue_cuda(self, t, img_offset, capacity):
        block, out = self._buffers(capacity)
        o = _lib.struct("mhmr_outputs", **t)
        s = self.stream.cuda_stream
        with torch.cuda.device(self.model.device):
            call("mhmr_pack_records", o, self.Pm, self.nb, self.V, img_offset, capacity, block, s)
            call("mhmr_allgather_records", self._comm, block, out, block.numel() * 4, s)
        return out

    # ---- public ------------------------------------------------------------------------------------
    def gather_async(self, t: dict, img_offset: int, count: int | None = None):
        """Enqueue pack + all-gather of the outputs `t` of a forward (max_persons-sized tensors).  `count` is
        only needed on the CPU path (the CUDA kernel reads it on the device)."""
        self.wait()
        if self.cuda:
            self.stream.wait_stream(torch.cuda.current_stream(self.model.device))
            out = self._enqueue_cuda(t, img_offset, self.capacity)
        else:
            block = pack_block_torch(t, int(count), img_offset, self.capacity, self.nb, self.V)
            out = torch.empty(self.world * block.numel(), dtype=block.dtype)
            dist.all_gather_into_tensor(out, block, group=self.group)
        self._pending = (t, img_offset, count, out)

    def wait(self):
        if self._pending is not None and self.cuda:
            self.stream.synchronize()

    def result(self):
        """(records [P_total, R] of all ranks in global (b, y, x) order, per-rank counts)."""
        assert self._pending is not None, "no gather in flight"
        t, img_offset, count, out = self._pending
        self.wait()
        detected, packed, recs = split_blocks(out, self.world, self.capacity, self.R)
        if max(detected) > self.capacity:  # rare: a rank overflowed the compact block -> one full-size round
            if max(detected) > self.Pm:
                raise RuntimeError(f"a rank detected {max(detected)} persons > max_persons {self.Pm}")
            if self.cuda:
                self.stream.wait_stream(torch.cuda.current_stream(self.model.device))
                out = self._enqueue_cuda(t, img_offset, self.Pm)
                self.stream.synchronize()
            else:
                block = pack_block_torch(t, int(count), img_offset, self.Pm, self.nb, self.V)
                out = torch.empty(self.world * block.numel(), dtype=block.dtype)
                dist.all_gather_into_tensor(out, block, group=self.group)
            detected, packed, recs = split_blocks(out, self.world, self.Pm, self.R)
        self._pending = None
        return recs.clone(), detected

    def close(self):
        if self._comm is not None:
            self.wait()
            _lib.load().mhmr_comm_destroy(self._comm)
            self._comm = None


class ShardedModel:
    """Runs `model` (a multihmr_b200.Model on this rank's GPU) on this rank's contiguous image shard of a
    global batch and all-gathers the persons."""

    def __init__(self, model, group=None, capacity=None):
        self.model, self.group = model, group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self.gather = RecordGather(model, self.rank, self.world, group, capacity)

    def forward(self, x_global, K_global, det_thresh=0.3, nms_kernel_size=3):
        lo, hi = shard_range(x_global.shape[0], self.world, self.rank)
        assert hi > lo, "every rank needs at least one image (the engine has no empty-batch forward)"
        t, P = self.model.forward_raw(x_global[lo:hi], K_global[lo:hi], det_thresh=det_thresh,
                                      nms_kernel_size=nms_kernel_size)
        self.gather.gather_async(t, lo, P)
        return self.gather.result()

    __call__ = forward
