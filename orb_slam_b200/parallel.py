"""Multi-GPU plumbing (torch.distributed; NCCL on the GPUs, gloo in CPU tests).

The extract path shards by frame/camera with no data-path collective (SURVEY.md 8e).  The only exchange step
is cross-frame matching between ranks (BASELINE config 4: one camera per GPU, cross-camera
SearchForInitialization): every rank contributes one fixed-capacity block
    [count | nfeatures x 28 B keypoints | nfeatures x 32 B descriptors]
and receives all blocks with a single all-gather (NVLink 5 / NVSwitch: ~0.1 MB per rank, latency-bound).
"""
import numpy as np

KP_BYTES = 28
DESC_BYTES = 32


def shard_range(n_items, world, rank):
    """Contiguous shard [lo, hi) of n_items for `rank` (keyframe DB rows, frames of a sequence)."""
    base, rem = divmod(n_items, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def block_bytes(nfeatures):
    return 16 + nfeatures * (KP_BYTES + DESC_BYTES)


def pack_block(torch, kps_u8, desc_u8, count, nfeatures, device):
    """kps_u8: [nfeatures, 28] uint8 tensor, desc_u8: [nfeatures, 32] uint8 tensor (device or cpu)."""
    blk = torch.zeros(block_bytes(nfeatures), dtype=torch.uint8, device=device)
    hdr = torch.tensor([int(count), nfeatures, 0, 0], dtype=torch.int32, device=device).view(torch.uint8)
    blk[:16] = hdr
    blk[16:16 + nfeatures * KP_BYTES] = kps_u8.reshape(-1)
    blk[16 + nfeatures * KP_BYTES:] = desc_u8.reshape(-1)
    return blk


def allgather_blocks(torch, dist, blk):
    """One all-gather of every rank's block; returns a [world, block_bytes] uint8 tensor."""
    world = dist.get_world_size() if dist.is_initialized() else 1
    out = torch.empty((world, blk.numel()), dtype=torch.uint8, device=blk.device)
    if world == 1:
        out[0] = blk
    else:
        dist.all_gather_into_tensor(out.view(-1), blk)
    return out


def unpack_block(row_u8_np, kp_dtype):
    """row: numpy uint8 [block_bytes] -> (kps[count], desc[count, 32])"""
    count, nfeatures = np.frombuffer(row_u8_np[:8].tobytes(), np.int32)
    kps = np.frombuffer(row_u8_np[16:16 + nfeatures * KP_BYTES].tobytes(), kp_dtype)[:count]
    desc = np.frombuffer(row_u8_np[16 + nfeatures * KP_BYTES:16 + nfeatures * (KP_BYTES + DESC_BYTES)].tobytes(),
                         np.uint8).reshape(nfeatures, 32)[:count]
    return kps, desc


def reduce_timing(torch, dist, ms, counts, device):
    """Bench contract: time = MAX over ranks, units = SUM over ranks."""
    t = torch.tensor([float(ms)], dtype=torch.float64, device=device)
    k = torch.tensor([float(c) for c in counts], dtype=torch.float64, device=device)
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        dist.all_reduce(k, op=dist.ReduceOp.SUM)
    return float(t[0]), [float(x) for x in k]
