"""GPU tests of the multi-GPU entry points (include/orbfe_comm.h) that make sense on ONE device: device-resident
SearchForInitialization (the matcher of config 4) against the oracle, and the rig exchange / sharded sweep with world = 1
(the peer table then holds only this rank: same kernels, same flags protocol).  The N > 1 runs are tools/multi_gpu.py under
torchrun; the host-side sharding logic is covered on CPU by tests/test_parallel_gloo.py."""
import numpy as np
import pytest

import oracle as O
import orb_slam_b200 as fe
from orb_slam_b200 import matching as M, comm as CM
from orb_slam_b200.synth import textured_frame, shifted_frame, random_descriptors

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("W,H,nf,ori,nnr", [(640, 480, 1000, True, 0.9), (1280, 720, 2000, True, 0.9), (1280, 720, 2000, False, 0.7)])
def test_device_search_for_initialization(gpu_required, W, H, nf, ori, nnr):
    """M8 in the fused kernel (MODE 2): several (F1, F2) pairs per launch incl. a frame against itself, the re-assignment rule,
    the rotation histogram with stale entries, the vbPrevMatched update; a second round with the updated positions."""
    import torch
    base = textured_frame(W, H, seed=71)
    imgs = [base, shifted_frame(base, 12, 4, seed=2), shifted_frame(base, -9, 6, seed=3), shifted_frame(base, 30, -14, seed=4)]
    ex = fe.ORBextractor(nf, 1.2, 8)
    kps, desc, cnt = ex.extract_batch(np.stack(imgs))
    ex.close()
    cnt = cnt.copy()
    cnt[2] -= 57                      # different counts per frame
    pairs = [(0, 1), (1, 0), (2, 3), (0, 3), (1, 1)]
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d_kps, d_desc, d_cnt = t(kps.view(np.uint8).reshape(len(imgs), nf, 28)), t(desc), t(cnt)
    d_f1, d_f2 = t(np.array([p[0] for p in pairs], np.int32)), t(np.array([p[1] for p in pairs], np.int32))
    prev = np.zeros((len(pairs), nf, 2), np.float32)
    for j, (a, b) in enumerate(pairs):
        prev[j, :, 0], prev[j, :, 1] = kps[a]["x"], kps[a]["y"]
    d_prev = t(prev)
    d_m12 = torch.full((len(pairs), nf), -7, dtype=torch.int32, device=dev)
    d_nm = torch.zeros(len(pairs), dtype=torch.int32, device=dev)
    m = fe.ORBmatcher(nnr, ori)
    prev_o = [prev[j, :cnt[a]].copy() for j, (a, b) in enumerate(pairs)]
    total = 0
    for rnd in range(2):
        M.search_for_initialization_device(m, len(pairs), d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), nf, d_f1.data_ptr(),
                                           d_f2.data_ptr(), d_prev.data_ptr(), W, H, 100, d_m12.data_ptr(), d_nm.data_ptr())
        m.sync()
        m12, nm, pv = d_m12.cpu().numpy(), d_nm.cpu().numpy(), d_prev.cpu().numpy()
        for j, (a, b) in enumerate(pairs):
            o1 = O.OracleFrame(kps[a][:cnt[a]], desc[a][:cnt[a]], W, H)
            o2 = O.OracleFrame(kps[b][:cnt[b]], desc[b][:cnt[b]], W, H)
            n_o, m_o, p_o = O.search_for_initialization(o1, o2, prev_o[j], 100, nnratio=nnr, check_orientation=ori)
            assert nm[j] == n_o, (rnd, j, nm[j], n_o)
            assert np.array_equal(m12[j, :cnt[a]], m_o), (rnd, j)
            assert np.array_equal(pv[j, :cnt[a]], p_o), (rnd, j)
            prev_o[j] = p_o
            total += n_o
    assert total > 200
    m.close()


def test_rig_exchange_and_sharded_sweep_world1(gpu_required):
    """World of one rank: the fused exchange (descriptor kernel -> gather buffer + epoch flag, wait, release; several epochs so
    that both buffer halves and the release wait are exercised) returns exactly what a plain extract returns; the sharded
    sweep degenerates to the plain sweep."""
    import torch
    import torch.distributed as dist
    W, H, nf, T = 1280, 720, 2000, 3
    frames = np.stack([textured_frame(W, H, seed=80 + i) for i in range(T)])
    dev = torch.device("cuda", 0)
    d_frames = torch.from_numpy(frames).to(dev)
    ex = fe.ORBextractor(nf, 1.2, 8)
    comm = CM.Comm.create(torch, dist, 0)
    assert comm.world == 1 and CM.nccl_version() >= 20000
    x = CM.RigExchange(comm, nf, T)
    d_kps = torch.zeros((T, nf, 28), dtype=torch.uint8, device=dev)
    d_desc = torch.zeros((T, nf, 32), dtype=torch.uint8, device=dev)
    d_cnt = torch.zeros((T,), dtype=torch.int32, device=dev)
    ex.extract_batch_device(d_frames.data_ptr(), W, H, W, W * H, T, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr())
    ex.sync()
    import sys, os
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    from multi_gpu import _as_tensor
    for epoch in range(5):
        x.extract(ex, d_frames.data_ptr(), W, H, W, W * H)
        x.wait()
        a, b, c = x.buffers()
        gk = _as_tensor(torch, a, (T, nf, 28), dev).clone()
        gd = _as_tensor(torch, b, (T, nf, 32), dev).clone()
        gc = _as_tensor(torch, c, (T,), dev, torch.int32).clone()
        x.release()
        x.check()
        assert torch.equal(gc, d_cnt) and torch.equal(gk, d_kps) and torch.equal(gd, d_desc), epoch
    assert x.bytes_pushed() == 0
    # the exchange-aware matcher call (waits for the epoch inside the kernel, releases it at its end) == the plain device call
    mm = fe.ORBmatcher(0.9, True)
    f1 = torch.tensor([0, 1], dtype=torch.int32, device=dev); f2 = torch.tensor([1, 2], dtype=torch.int32, device=dev)
    res = []
    for use_exchange in (False, True):
        prev = d_kps.view(torch.float32).view(T, nf, 7)[:2, :, 0:2].contiguous()
        m12 = torch.full((2, nf), -5, dtype=torch.int32, device=dev); nm = torch.zeros(2, dtype=torch.int32, device=dev)
        if use_exchange:
            x.extract(ex, d_frames.data_ptr(), W, H, W, W * H)
            x.search_for_initialization(mm, 2, f1.data_ptr(), f2.data_ptr(), prev.data_ptr(), W, H, 100, m12.data_ptr(), nm.data_ptr())
            x.check()
        else:
            M.search_for_initialization_device(mm, 2, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), nf, f1.data_ptr(), f2.data_ptr(),
                                               prev.data_ptr(), W, H, 100, m12.data_ptr(), nm.data_ptr())
            mm.sync()
        res.append((m12.cpu().numpy(), nm.cpu().numpy(), prev.cpu().numpy()))
    assert all(np.array_equal(a, b) for a, b in zip(res[0], res[1]))
    mm.close()
    # plain all-gather of one rank = copy
    g2 = torch.zeros_like(d_kps); gd2 = torch.zeros_like(d_desc); gc2 = torch.zeros_like(d_cnt)
    comm.allgather_desc(d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), nf, T, g2.data_ptr(), gd2.data_ptr(), gc2.data_ptr())
    comm.sync()
    assert torch.equal(g2, d_kps) and torch.equal(gd2, d_desc) and torch.equal(gc2, d_cnt)
    # sharded sweep with one shard
    nq, per, ng = 256, 500, 12
    q, db = random_descriptors(nq, 1), random_descriptors(ng * per, 2)
    m = fe.ORBmatcher()
    dq, ddb = torch.from_numpy(q).to(dev), torch.from_numpy(db).to(dev)
    best = torch.zeros((ng, nq), dtype=torch.uint16, device=dev)
    idx = torch.zeros((ng, nq), dtype=torch.int32, device=dev)
    second = torch.zeros((ng, nq), dtype=torch.uint16, device=dev)
    scratch = torch.zeros((2 * ng * nq * 8,), dtype=torch.uint8, device=dev)
    comm.knn2_sweep_sharded(m, dq.data_ptr(), nq, 0, ddb.data_ptr(), ng, per, best.data_ptr(), idx.data_ptr(), second.data_ptr(), scratch.data_ptr())
    comm.sync()
    for g in (0, 5, 11):
        bd, bi, sd = O.knn2(q, db[g * per:(g + 1) * per])
        assert np.array_equal(best[g].cpu().numpy(), bd) and np.array_equal(idx[g].cpu().numpy(), bi)
        assert np.array_equal(second[g].cpu().numpy(), np.minimum(sd, 65535))
    assert CM.shard_range(10, 4, 1) == (3, 6) and CM.shard_range(10000, 8, 7) == (8750, 10000)
    m.close(); x.close(); comm.close(); ex.close()
