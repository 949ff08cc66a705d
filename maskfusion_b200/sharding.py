"""Object-sharded MaskFusion: one process per GPU, object Models partitioned over the ranks (SURVEY 8e).

Per frame the ranks exchange exactly what couples the models in the reference:

  frame in          rgb + depth + instance mask + class ids, broadcast from the loader rank     (MaskFusion.cpp:212-217)
  poses             every tracked model's pose / last transform, all-gather                      (MaskFusion.cpp:257-276)
  ID projection     64-bit (depth bits << 32 | model index << 26 | surfel) keys, all-reduce MIN  (GlobalProjection.cpp:66-95)
  masks             with a detector rank (attachDetector), on detector frames: that rank's frame mask + header, broadcast

Everything after the merged key image (segmentation, mask<->model voting, spawn decision, inactivation) is a
deterministic function of replicated inputs and is evaluated on every rank; the surfel passes (index map,
association, fusion, clean, splat) run only on the rank that holds the model's store.  On the GPU box the three
exchanges are NCCL calls issued INSIDE the library (mf_shard_process_frame, csrc/mf_sched.cu); this file bootstraps the
communicator and keeps a host-staged transport over the phase-split ABI for backends without NCCL (gloo: how the
path is tested on one GPU or none).

The helpers at module level are device-agnostic and are what tests/test_cpu_sharding.py exercises over gloo.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import api

_SIGN = -(2 ** 63)
MAX_MODELS = 64
MAX_CLASSES = 256


# ------------------------------------------------------------------------------------------------------------
# device-agnostic plumbing (torch tensors, any backend)
# ------------------------------------------------------------------------------------------------------------
def frame_packet_bytes(W: int, H: int) -> int:
    """rgb (3P) | depth f32 (4P) | mask u8 (P) | header int64[2] = (timestamp, nClasses) | classIDs int32[256]"""
    P = W * H
    return 8 * P + 16 + 4 * MAX_CLASSES


def pack_frame(buf, W, H, rgb, depth, mask, timestamp, classIDs):
    """loader rank: fill the broadcast packet (a uint8 torch tensor of frame_packet_bytes) from numpy inputs"""
    import torch
    P = W * H
    n = 0 if classIDs is None else len(classIDs)
    if n > MAX_CLASSES:
        raise api.MFError("more than 256 mask labels")
    host = np.zeros(frame_packet_bytes(W, H), np.uint8)
    host[0:3 * P] = np.ascontiguousarray(rgb, np.uint8).reshape(-1)
    host[3 * P:7 * P] = np.ascontiguousarray(depth, np.float32).reshape(-1).view(np.uint8)
    if mask is not None:
        host[7 * P:8 * P] = np.ascontiguousarray(mask, np.uint8).reshape(-1)
    host[8 * P:8 * P + 16] = np.array([int(timestamp), n if mask is not None else -1], np.int64).view(np.uint8)
    if n:
        host[8 * P + 16:8 * P + 16 + 4 * n] = np.ascontiguousarray(classIDs, np.int32).view(np.uint8)
    buf.copy_(torch.from_numpy(host), non_blocking=False)


def unpack_header(buf, W, H):
    """-> (timestamp, classIDs or None); one small device->host read"""
    P = W * H
    tail = buf[8 * P:].cpu().numpy()
    ts, n = (int(v) for v in tail[:16].view(np.int64))
    if n < 0:
        return ts, None
    return ts, tail[16:16 + 4 * n].view(np.int32).copy()


def allreduce_min_u64(keys_i64, group=None):
    """unsigned 64-bit MIN all-reduce of a tensor that holds uint64 bit patterns in int64 storage.
    Flipping the top bit maps unsigned order onto signed order (the empty key 0xFFFF.. must stay the maximum)."""
    import torch
    import torch.distributed as dist
    sign = torch.tensor(_SIGN, dtype=torch.int64, device=keys_i64.device)
    keys_i64.bitwise_xor_(sign)
    dist.all_reduce(keys_i64, op=dist.ReduceOp.MIN, group=group)
    keys_i64.bitwise_xor_(sign)
    return keys_i64


def gather_rows(local_rows, group=None):
    """all-gather of a [nModels, 32] float32 table -> [world, nModels, 32] (bit-exact: no arithmetic on the payload)"""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group)
    flat = local_rows.contiguous().view(-1)
    out = torch.empty(world * flat.numel(), dtype=flat.dtype, device=flat.device)
    dist.all_gather_into_tensor(out, flat, group=group)
    return out.view((world,) + tuple(local_rows.shape))


def pick_owner(loads) -> int:
    """placement of a new model (host rule shared with the library: mf_shard_pick_owner)"""
    a = np.ascontiguousarray(loads, np.int64)
    r = api.load_library().mf_shard_pick_owner(a.ctypes.data_as(C.c_void_p), int(a.shape[0]))
    if r < 0:
        raise api.MFError("pick_owner: bad arguments")
    return r


class _DevPtr:
    """expose a raw device pointer to torch through __cuda_array_interface__"""

    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (int(ptr), False), "version": 2}


# ------------------------------------------------------------------------------------------------------------
class ShardedMaskFusion:
    """MaskFusion with the object Models sharded over the ranks of a torch.distributed group.

    Every rank constructs it with the same config and calls processFrame every frame; only `src` (rank 0) needs real
    inputs.  Poses, ids, classes and pose logs of ALL models are available on every rank; surfel read-backs only
    on the owner (`owner(i)`).

    Two transports:
      * NCCL (one GPU per rank): the exchange lives INSIDE the library.  This class only bootstraps the communicator -- rank 0
        draws the NCCL unique id (mf_shard_unique_id), torch.distributed carries the 128 bytes to the other ranks,
        mf_shard_comm_init creates the communicator on the context's device -- and then forwards every frame to
        mf_shard_process_frame: broadcast of the frame packet, all-gather of the pose rows and the 64-bit MIN all-reduce of the
        ID-projection keys are NCCL calls issued by the library on the context's stream, with no host synchronisation in the frame.
      * anything else (gloo in the tests; all ranks may share one GPU): the transport-agnostic phase calls of the C ABI with the
        rows and keys staged through the host by the helpers above."""

    def __init__(self, cfg: api.Config, device: int = 0, group=None, src: int = 0):
        import torch
        import torch.distributed as dist
        if not dist.is_initialized():
            raise api.MFError("ShardedMaskFusion needs an initialised torch.distributed process group")
        if src != 0:
            raise api.MFError("the loader rank is rank 0 (it also owns the background model)")
        self.torch, self.dist, self.group, self.src = torch, dist, group, src
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        self.on_nccl = dist.get_backend(group) == "nccl"
        self.dev = torch.device("cuda", device)
        torch.cuda.set_device(self.dev)
        # one explicit stream for the kernels AND (gloo path) the staging ops: torch's default stream has the NULL handle, which
        # mf_create reads as "make a private non-blocking stream" -- torch ops on the default stream would then race with the kernels
        self.stream = torch.cuda.Stream(self.dev)
        self.mf = api.MaskFusion(cfg, device=device, stream=self.stream.cuda_stream)
        self.L, self.h = self.mf.L, self.mf.h
        self.W, self.H = cfg.width, cfg.height
        self.P = self.W * self.H
        self.bytes_collective = 0
        self.det_rank = -1
        if self.on_nccl:
            uid = torch.zeros(128, dtype=torch.uint8)
            if self.rank == 0:
                b = (C.c_uint8 * 128)()
                self.mf._ck(self.L.mf_shard_unique_id(b))
                uid = torch.frombuffer(bytearray(b), dtype=torch.uint8).clone()
            uid = uid.to(self.dev)
            dist.broadcast(uid, src=0, group=group)                      # the only use of torch's collectives: 128 bytes, once
            raw = (C.c_uint8 * 128).from_buffer_copy(bytes(uid.cpu().numpy().tobytes()))
            self.mf._ck(self.L.mf_shard_comm_init(self.h, raw, self.rank, self.world))
        else:
            self.mf._ck(self.L.mf_shard_configure(self.h, self.rank, self.world))
            with torch.cuda.stream(self.stream):
                self.packet = torch.zeros(frame_packet_bytes(self.W, self.H), dtype=torch.uint8, device=self.dev)
            self.packet_host = torch.zeros(frame_packet_bytes(self.W, self.H), dtype=torch.uint8).pin_memory()
            self.keys = None
            self.rows = np.zeros((MAX_MODELS, 32), np.float32)

    # -- gloo path: collectives staged through the host --
    def _broadcast_packet(self):
        self.packet_host.copy_(self.packet)
        self.dist.broadcast(self.packet_host, src=self.src, group=self.group)
        self.packet.copy_(self.packet_host)
        self.bytes_collective += self.packet.numel()

    def _exchange_poses(self):
        g = gather_rows(self.torch.from_numpy(self.rows), self.group)
        self.bytes_collective += g.numel() * 4
        return np.ascontiguousarray(g.numpy())

    def _merge_keys(self):
        if self.keys is None:
            ptr = self.L.mf_shard_projection_keys(self.h)
            self.keys = self.torch.as_tensor(_DevPtr(ptr, self.P, "<i8"), device=self.dev)
        k = self.keys.cpu()
        allreduce_min_u64(k, self.group)
        self.keys.copy_(k)
        self.bytes_collective += self.P * 8

    def _exchange_masks(self):
        """detector frames: the detector rank's frame mask | header to every rank (mf_shard_frame_masks says when and where)"""
        ptr, n = C.c_void_p(), C.c_size_t()
        if not self.mf._ck(self.L.mf_shard_frame_masks(self.h, C.byref(ptr), C.byref(n))):
            return
        tail = self.torch.as_tensor(_DevPtr(ptr.value, n.value, "|u1"), device=self.dev)
        host = tail.cpu()
        src = self.det_rank if self.group is None else self.dist.get_global_rank(self.group, self.det_rank)
        self.dist.broadcast(host, src=src, group=self.group)
        tail.copy_(host)
        self.bytes_collective += n.value

    # -- one frame --
    def processFrame(self, rgb=None, depth=None, timestamp: int = 0, mask=None, classIDs=None, weightMultiplier: float = 1.0):
        if self.on_nccl:
            return self._process_frame_nccl(rgb, depth, timestamp, mask, classIDs, weightMultiplier)
        with self.torch.cuda.stream(self.stream):            # every torch op below is ordered with the kernels on self.stream
            return self._process_frame_staged(rgb, depth, timestamp, mask, classIDs, weightMultiplier)

    def _process_frame_nccl(self, rgb, depth, timestamp, mask, classIDs, weightMultiplier):
        ck, L, h = self.mf._ck, self.L, self.h
        if self.rank == 0:
            rgb = np.ascontiguousarray(rgb, np.uint8); depth = np.ascontiguousarray(depth, np.float32)
            m = None if mask is None else np.ascontiguousarray(mask, np.uint8)
            c = None if classIDs is None else np.ascontiguousarray(classIDs, np.int32)
            ck(L.mf_shard_process_frame(h, rgb.ctypes.data_as(C.c_void_p), depth.ctypes.data_as(C.c_void_p), int(timestamp),
                                        None if m is None else m.ctypes.data_as(C.c_void_p), None if c is None else c.ctypes.data_as(C.c_void_p),
                                        0 if c is None else int(c.shape[0]), float(weightMultiplier), 0))
        else:
            ck(L.mf_shard_process_frame(h, None, None, 0, None, None, 0, float(weightMultiplier), 0))
        return False

    def processFramePtr(self, rgb_ptr, depth_ptr, timestamp, mask_ptr, cls_ptr, n_cls, on_device=False, weightMultiplier=1.0):
        """NCCL path with raw pointers (pinned host or device memory of rank 0; class ids always on the host): what bench.py times;
        the arguments are ignored on the other ranks"""
        self.mf._ck(self.L.mf_shard_process_frame(self.h, C.c_void_p(rgb_ptr), C.c_void_p(depth_ptr), int(timestamp), C.c_void_p(mask_ptr),
                                                  C.c_void_p(cls_ptr), int(n_cls), float(weightMultiplier), int(bool(on_device))))

    def _process_frame_staged(self, rgb, depth, timestamp, mask, classIDs, weightMultiplier):
        ck, L, h, P = self.mf._ck, self.L, self.h, self.P
        if self.rank == self.src:
            pack_frame(self.packet, self.W, self.H, rgb, depth, mask, timestamp, classIDs)
        self._broadcast_packet()
        ts, classes = unpack_header(self.packet, self.W, self.H)
        base = self.packet.data_ptr()
        if classes is not None:
            ck(L.mf_set_frame_classes(h, classes.ctypes.data_as(C.c_void_p), int(classes.shape[0])))
        else:
            ck(L.mf_set_frame_classes(h, None, 0))
        ck(L.mf_shard_frame_begin(h, C.c_void_p(base), C.c_void_p(base + 3 * P), ts, C.c_void_p(base + 7 * P) if classes is not None else None, 1))
        if self.mf.getTick() > 1:
            ck(L.mf_shard_get_poses(h, self.rows.ctypes.data_as(C.c_void_p), MAX_MODELS))
            gathered = self._exchange_poses()
            ck(L.mf_shard_set_poses(h, gathered.ctypes.data_as(C.c_void_p)))
        ck(L.mf_shard_project(h))
        if self.mf.cfg.enableMultipleModels and self.mf.getTick() > 1:
            self._merge_keys()
        self._exchange_masks()
        ck(L.mf_shard_frame_end(h, float(weightMultiplier)))
        return False

    # -- Mask R-CNN on one rank --
    def attachDetector(self, detector, every_k: int = 1, rank: int | None = None):
        """every rank, between the same frames: the detector runs on `rank` (default world - 1: rank 0 already carries the loader and the
        background model) every k-th tracking frame, and its masks reach every rank.  `detector` is ignored, and may be None, on the
        other ranks.  The shards then compute what one MaskFusion with attachDetector(detector, every_k) computes."""
        r = self.world - 1 if rank is None else int(rank)
        d = C.c_void_p(detector.h) if detector is not None and self.rank == r else None
        self.mf._ck(self.L.mf_shard_attach_detector(self.h, d, int(every_k), r))
        self.det_rank = r

    def detachDetector(self):
        """every rank, between the same frames; the detector rank first waits for the last hand-off"""
        self.mf._ck(self.L.mf_shard_attach_detector(self.h, None, 0, -1))
        self.det_rank = -1

    def frameMasks(self):
        """-> (mask, class ids) that segmentation read on the last frame: the same on every rank"""
        return self.mf.frameMasks()

    def stats(self):
        """-> dict(bytes, calls, nranks, nccl_version): collectives issued by the library (NCCL path) or by this class (staged path)"""
        out = (C.c_int64 * 4)()
        self.mf._ck(self.L.mf_shard_stats(self.h, out))
        if not self.on_nccl:
            return {"bytes": int(self.bytes_collective), "calls": None, "nranks": self.world, "nccl_version": 0, "transport": "host-staged"}
        return {"bytes": int(out[0]), "calls": int(out[1]), "nranks": int(out[2]), "nccl_version": int(out[3]), "transport": "nccl (in-library)"}

    # -- replicated queries --
    def owner(self, i: int) -> int:
        return self.mf._ck(self.L.mf_model_owner(self.h, i))

    def models(self):
        return self.mf.getModels()

    def close(self):
        self.mf.close()
