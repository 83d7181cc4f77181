"""Frame-level data parallelism: one process per GPU, frames are independent units
(SURVEY.md §8e), frame i -> rank i mod W (the shape of the reference's dead
DistEvalHook, mmdet/core/evaluation/eval_hooks.py:72), one NCCL all_gather of the
fixed-size result tensors at the end of a shard.  No collective inside a frame."""
import os

import torch
import torch.distributed as dist


def init_from_env(backend=None):
    """torchrun-style env (RANK / WORLD_SIZE / LOCAL_RANK / MASTER_*).  Returns (rank, world, local_rank)."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        kw = {}
        if backend == "nccl":
            torch.cuda.set_device(local)
            kw["device_id"] = torch.device("cuda", local)      # eager communicator creation, no lazy first-use cost
        dist.init_process_group(backend=backend, rank=rank, world_size=world, **kw)
    return rank, world, local


def shard_frames(n_frames, rank, world):
    """Indices of the frames this rank owns."""
    return list(range(rank, n_frames, world))


class DetectionGather:
    """The shard's single exchange step (SURVEY.md section 8e): ONE all_gather_into_tensor of the fixed-size result
    block [det | ndet] per rank into a pre-allocated buffer (the reference pickles per-rank result lists to a shared
    file system, mmdet/core/evaluation/eval_hooks.py:92-106).  ``warm()`` runs the collective once so that
    communicator / channel set-up is not inside anybody's timed region.  ``width``: float32 words per row (9 for the
    detections; the KITTI rows of ops.kitti_format are 14 float64 = 28 words, passed as ``rows.view(torch.float32)``)."""

    def __init__(self, frames_local, det_cap, device, width=9):
        self.F, self.cap, self.device, self.width = int(frames_local), int(det_cap), device, int(width)
        self.world = dist.get_world_size() if (dist.is_available() and dist.is_initialized()) else 1
        self.row = self.F * self.cap * self.width + self.F         # floats per rank: row block + counts (as f32 bits)
        self.send = torch.zeros((self.row,), dtype=torch.float32, device=device)
        self.recv = torch.zeros((self.world * self.row,), dtype=torch.float32, device=device)

    def warm(self):
        self(torch.zeros((self.F, self.cap, self.width), dtype=torch.float32, device=self.device),
             torch.zeros((self.F,), dtype=torch.int32, device=self.device))
        if self.device.type == "cuda":
            torch.cuda.synchronize(self.device)

    def __call__(self, det, ndet):
        """det [F, cap, width] f32, ndet [F] i32 -> det [W, F, cap, width], ndet [W, F] on every rank
        (frame (r, j) is global frame j*W + r)."""
        n = self.F * self.cap * self.width
        self.send[:n].copy_(det.reshape(-1))
        self.send[n:].copy_(ndet.view(torch.float32) if ndet.dtype == torch.int32 else ndet.int().view(torch.float32))
        if self.world == 1:
            self.recv.copy_(self.send)
        else:
            dist.all_gather_into_tensor(self.recv, self.send)
        blocks = self.recv.view(self.world, self.row)
        return (blocks[:, :n].reshape(self.world, self.F, self.cap, self.width),
                blocks[:, n:].contiguous().view(torch.int32))


def gather_detections(det, ndet):
    """One-shot form of DetectionGather (allocates; use the class on a hot path)."""
    return DetectionGather(det.shape[0], det.shape[1], det.device, width=det.shape[2])(det, ndet)


def interleave(det_all, ndet_all):
    """[W, F, cap, width] -> global frame order [W*F, cap, width] (frame j*W + r)."""
    W, Fl = det_all.shape[0], det_all.shape[1]
    return (det_all.permute(1, 0, 2, 3).reshape(W * Fl, *det_all.shape[2:]),
            ndet_all.permute(1, 0).reshape(W * Fl))


def max_over_ranks(value, device):
    t = torch.tensor([float(value)], dtype=torch.float64, device=device)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def barrier():
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.barrier()
