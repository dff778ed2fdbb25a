"""Multi-GPU plumbing: frames are independent (SURVEY.md 8e), so a batch is
sharded over ranks with no data-path collective except ONE all-gather of the
fixed-shape pose tensor (+ n_valid packed into the same buffer).  Replaces the
reference's training-only single-process DataParallel
(models/data_parallel.py:10-84) on the inference path.

Tracking shards video SLOTS the same way (`slot_layout`): each rank steps its own slots and the per-frame exchange is
one all-gather of [slots/rank, max_tracks, CP_TRACK_RECORD] track records + n_tracks, a `PoseBuffer` with
K = max_tracks and R = CP_TRACK_RECORD.

`PoseBuffer` is the persistent buffer of that exchange: ONE flat fp32 tensor per rank,
    [ poses  b*K*R floats | n_valid  b int32 (same 4-byte cells) ]
whose two views are handed to `cp_infer` as its output pointers, so the kernels write the packed layout directly --
no concatenation / conversion kernel runs on the hot path.  The all-gather lands in a second persistent buffer
[world, b*K*R + b]; a device -> host copy (rank 0, or whoever asks) goes into pinned memory.
"""
import torch
import torch.distributed as dist

from . import _lib


def shard_range(n, rank, world):
    """Contiguous [start, stop) of frame indices owned by `rank` (sizes differ by at most one)."""
    base, rem = divmod(n, world)
    start = rank * base + min(rank, rem)
    return start, start + base + (1 if rank < rem else 0)


def slot_layout(slots, world):
    """Tracking slots over `world` ranks: rank r owns slots shard_range(slots, r, world) and every rank gathers the same
    number of rows, b = ceil(slots / world) (a rank with fewer slots leaves its last row empty).  Returns (b, order):
    order[i] is the row of slot i in the gathered [world * b] records."""
    b = -(-int(slots) // int(world))
    order = []
    for r in range(world):
        lo, hi = shard_range(slots, r, world)
        order += [r * b + k for k in range(hi - lo)]
    return b, order


class PoseBuffer(object):
    def __init__(self, batch, K, device, world=1, R=_lib.CP_POSE_RECORD, pin=True):
        self.b, self.K, self.R, self.world = int(batch), int(K), int(R), int(world)
        self.n_pose = self.b * self.K * self.R
        self.row = self.n_pose + self.b
        self.flat = torch.zeros((self.row,), dtype=torch.float32, device=device)
        self.poses = self.flat[:self.n_pose].view(self.b, self.K, self.R)            # cp_infer writes here
        self.n_valid = self.flat[self.n_pose:].view(torch.int32)                     # ... and here
        self.gathered = (torch.zeros((self.world, self.row), dtype=torch.float32, device=device)
                         if self.world > 1 else self.flat.view(1, self.row))
        pinned = pin and torch.device(device).type == "cuda"
        self.host = torch.zeros((self.world, self.row), dtype=torch.float32, pin_memory=pinned)
        self._evt = torch.cuda.Event() if torch.device(device).type == "cuda" else None

    def all_gather(self, group=None):
        """The one collective of the data path.  No-op for a single rank."""
        if self.world > 1:
            dist.all_gather_into_tensor(self.gathered.view(-1), self.flat, group=group)
        return self.gathered

    def views(self, buf):
        """[world, row] buffer (device or host) -> (poses [world*b, K, R], n_valid [world*b])."""
        poses = buf[:, :self.n_pose].reshape(self.world * self.b, self.K, self.R)     # a copy only when world > 1
        n_valid = buf[:, self.n_pose:].contiguous().view(torch.int32).reshape(-1)
        return poses, n_valid

    def to_host(self, sync=True):
        """Asynchronous D2H of the gathered records into the pinned host buffer (one contiguous copy)."""
        self.host.copy_(self.gathered, non_blocking=True)
        if self._evt is not None:
            self._evt.record()
            if sync:
                self._evt.synchronize()
        return self.host

    def host_views(self):
        h = self.host.numpy()
        poses = h[:, :self.n_pose].reshape(self.world * self.b, self.K, self.R)
        n_valid = h[:, self.n_pose:].copy().view("int32").reshape(-1)
        return poses, n_valid


# ---- functional form kept for callers that hold separate tensors (and the gloo CPU test) ------------------------------
def pack(poses, n_valid):
    """[b,K,R] fp32 + [b] int32 -> flat [b*K*R + b] fp32 cells (n_valid bit-cast, not converted)."""
    return torch.cat([poses.reshape(-1), n_valid.to(torch.int32).contiguous().view(torch.float32).reshape(-1)])


def unpack(flat, b, K, R=_lib.CP_POSE_RECORD):
    return flat[:b * K * R].view(b, K, R), flat[b * K * R:].contiguous().view(torch.int32)


def all_gather_poses(poses, n_valid, group=None):
    """One collective: every rank receives the pose records of the whole batch, in rank order.
    Requires equal per-rank batch (the weak-scaling configuration).  Hot paths use `PoseBuffer` instead."""
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return poses, n_valid
    world = dist.get_world_size(group)
    b, K, R = poses.shape
    local = pack(poses, n_valid)
    out = torch.empty((world, local.numel()), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out.view(-1), local, group=group)
    ps, ns = zip(*[unpack(out[r], b, K, R) for r in range(world)])
    return torch.cat(ps), torch.cat(ns)
