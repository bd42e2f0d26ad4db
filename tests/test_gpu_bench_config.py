"""GPU parity of SearchByProjection(Frame, Frame) (reference src/ORBmatcher.cc:1507-1620) at the BENCHMARKED configuration:
1920x1080, 2000 keypoints per frame, cap 2000, consecutive frames of a stream.  At this size the fused kernel loops
twice over the queries (2000 > 1024 threads) and its candidate entries may live in shared memory or in the per-pair
global scratch (match_kernels.cu `ent = T_total <= smem_entries ? s_ent : scratch`): both placements are forced here,
through the device-pointer entry point and through the host-view entry point, against the oracle."""
import os

import numpy as np
import pytest

import oracle as O
import orb_slam_b200 as fe
from orb_slam_b200 import matching as M
from orb_slam_b200.synth import textured_frame, shifted_frame

pytestmark = pytest.mark.gpu

W, H, NF = 1920, 1080, 2000
FX = FY = 1000.0
CX, CY, DEPTH = W / 2.0, H / 2.0, 5.0
NFRAMES = 9   # 8 consecutive pairs


def _tcw(dx, dy):
    T = np.zeros((3, 4), np.float32)
    T[0, 0] = T[1, 1] = T[2, 2] = 1
    T[0, 3], T[1, 3] = dx * DEPTH / FX, dy * DEPTH / FY
    return T


def _world(k):
    w = np.empty((len(k), 3), np.float32)
    w[:, 0] = (k["x"] - np.float32(CX)) / np.float32(FX) * np.float32(DEPTH)
    w[:, 1] = (k["y"] - np.float32(CY)) / np.float32(FY) * np.float32(DEPTH)
    w[:, 2] = DEPTH
    return w


@pytest.fixture(scope="module")
def stream(gpu_required):
    rng = np.random.default_rng(5)
    frames, shifts = [textured_frame(W, H, seed=77)], [(0, 0)]
    for i in range(1, NFRAMES):
        dx, dy = int(rng.integers(-6, 7)), int(rng.integers(-4, 5))
        frames.append(shifted_frame(frames[-1], dx, dy, seed=100 + i))
        shifts.append((dx, dy))
    ex = fe.ORBextractor(NF, 1.2, 8)
    kps, desc, cnt = ex.extract_batch(np.stack(frames))
    ex.close()
    assert list(cnt) == [NF] * NFRAMES
    # the extractor itself at this geometry: two of the frames against the oracle
    p = O.make_params(NF, 1.2, 8, 1, 20)
    for f in (0, NFRAMES - 1):
        rc, ok, od, _ = O.extract(p, frames[f])
        assert rc == 0 and np.array_equal(desc[f], od)
        for name in ("x", "y", "octave", "response"):
            assert np.array_equal(kps[f][name], ok[name]), name
    has = [(rng.random(NF) < 0.93).astype(np.uint8) for _ in range(NFRAMES)]
    outl = [(rng.random(NF) < 0.04).astype(np.uint8) for _ in range(NFRAMES)]
    pre = []
    for _ in range(NFRAMES):
        occ = np.full(NF, -1, np.int32)
        occ[rng.random(NF) < 0.03] = 11   # slots occupied on entry (ORBmatcher.cc:1562)
        pre.append(occ)
    return kps, desc, shifts, has, outl, pre


def _oracle(stream, th, ori):
    kps, desc, shifts, has, outl, pre = stream
    out = []
    for j in range(1, NFRAMES):
        fc = O.OracleFrame(kps[j], desc[j], W, H)
        fl = O.OracleFrame(kps[j - 1], desc[j - 1], W, H)
        out.append(O.search_by_projection_ff(fc, fl, has[j - 1], outl[j - 1], _world(kps[j - 1]), _tcw(*shifts[j]), FX, FY, CX, CY,
                                             th, ori, cur_mp=pre[j]))
    return out


@pytest.fixture(params=[0, 1], ids=["smem-entries", "global-scratch"])
def entry_placement(request):
    if request.param:
        os.environ["ORBFE_SBP_FORCE_SCRATCH"] = "1"
    yield request.param
    os.environ.pop("ORBFE_SBP_FORCE_SCRATCH", None)


@pytest.mark.parametrize("th,ori", [(15.0, True), (15.0, False), (40.0, True)])
def test_sbp_device_at_bench_config(stream, entry_placement, th, ori):
    """orbfe_search_by_projection_device: th=15 is Tracking.cc:565; th=40 multiplies the candidate lists by ~7 (the
    entries then exceed the shared-memory staging area by themselves)."""
    import torch
    kps, desc, shifts, has, outl, pre = stream
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    npairs = NFRAMES - 1
    world = np.stack([_world(kps[f]) for f in range(NFRAMES)])
    flags = np.stack([(has[f] & (1 - outl[f])).astype(np.uint8) for f in range(NFRAMES)])
    T = np.stack([_tcw(*shifts[j]) for j in range(1, NFRAMES)]).reshape(npairs, 12).astype(np.float32)
    d_kps, d_desc = t(kps.view(np.uint8).reshape(NFRAMES, NF, 28)), t(desc)
    d_cnt = t(np.full(NFRAMES, NF, np.int32))
    d_mp = t(np.stack(pre[1:]))
    d_nm = torch.zeros(npairs, dtype=torch.int32, device=dev)
    d_cur, d_last = t(np.arange(1, NFRAMES, dtype=np.int32)), t(np.arange(0, NFRAMES - 1, dtype=np.int32))
    d_world, d_flags, d_T = t(world), t(flags), t(T)
    torch.cuda.synchronize()
    m = fe.ORBmatcher(0.9, ori)
    M.search_by_projection_device(m, npairs, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), NF, d_cur.data_ptr(),
                                  d_last.data_ptr(), d_world.data_ptr(), d_flags.data_ptr(), d_T.data_ptr(), W, H, 1.2, 8,
                                  FX, FY, CX, CY, th, d_mp.data_ptr(), d_nm.data_ptr())
    m.sync()
    mp, nm = d_mp.cpu().numpy(), d_nm.cpu().numpy()
    ref = _oracle(stream, th, ori)
    tot = 0
    for j in range(npairs):
        assert nm[j] == ref[j][0], (j, nm[j], ref[j][0])
        assert np.array_equal(mp[j], ref[j][1]), j
        tot += ref[j][0]
    assert tot > 8 * 800   # the stream has true matches at this size too
    m.close()


def test_sbp_frames_at_bench_config(stream, entry_placement):
    """orbfe_search_by_projection_frames (the call behind ORBmatcher::SearchByProjection(Frame&, const Frame&, float))
    with host views, eight pairs per call."""
    kps, desc, shifts, has, outl, pre = stream
    views = [M.FrameView(kps[f], desc[f], W, H) for f in range(NFRAMES)]
    m = fe.ORBmatcher(0.9, True)
    nm, mp = M.search_by_projection_frames(m, views[1:], views[:-1], has[:-1], outl[:-1], [_world(kps[f]) for f in range(NFRAMES - 1)],
                                           [_tcw(*shifts[j]) for j in range(1, NFRAMES)], FX, FY, CX, CY, 15.0, cur_mp=pre[1:])
    ref = _oracle(stream, 15.0, True)
    for j in range(NFRAMES - 1):
        assert nm[j] == ref[j][0] and np.array_equal(mp[j], ref[j][1]), j
    m.close()


def test_stream_driver_equals_direct_calls_and_oracle(gpu_required):
    """bench.py's end-to-end pipeline (tools/e2e_driver.cpp on C++ threads: two extractor handles and two matcher handles
    alternating batches, frame views and synthetic map points built in C++) produces, for every frame of a small stream, the
    keypoints / descriptors of a direct orbfe_extract_batch call, and for every consecutive pair -- the pairs that straddle
    two batches included -- the match vector of the CPU oracle."""
    import torch
    from orb_slam_b200.stream_driver import StreamDriver
    w, h, nf, B, NB = 640, 480, 600, 4, 3
    fx = fy = 500.0
    cx, cy, depth, th = w / 2.0, h / 2.0, 4.0, 15.0
    rng = np.random.default_rng(9)
    frames, shifts = [textured_frame(w, h, seed=21)], [(0, 0)]
    for i in range(1, B * NB):
        dx, dy = int(rng.integers(-5, 6)), int(rng.integers(-3, 4))
        frames.append(shifted_frame(frames[-1], dx, dy, seed=300 + i))
        shifts.append((dx, dy))
    frames = np.stack(frames)

    def tcw(dx, dy):
        T = np.zeros((3, 4), np.float32)
        T[0, 0] = T[1, 1] = T[2, 2] = 1
        T[0, 3], T[1, 3] = dx * depth / fx, dy * depth / fy
        return T
    Tcws = np.stack([tcw(*s) for s in shifts]).reshape(-1, 12)
    h_frames = torch.from_numpy(frames).pin_memory()
    nex, nmatch = 2, 2
    bufs = [(torch.zeros((B, nf, 28), dtype=torch.uint8).pin_memory(), torch.zeros((B, nf, 32), dtype=torch.uint8).pin_memory(),
             torch.zeros((B,), dtype=torch.int32).pin_memory()) for _ in range(nex + nmatch)]
    drv = StreamDriver(w, h, nf, 8, 1.2, 20, B, NB, nex, nmatch, 0, fx, fy, cx, cy, depth, th, h_frames.data_ptr(), Tcws,
                       [b[0].data_ptr() for b in bufs], [b[1].data_ptr() for b in bufs], [b[2].data_ptr() for b in bufs])
    ex = fe.ORBextractor(nf, 1.2, 8)
    kps, desc, cnt = ex.extract_batch(frames)
    ex.close()

    def world(k):
        o = np.empty((len(k), 3), np.float32)
        o[:, 0] = (k["x"] - np.float32(cx)) / np.float32(fx) * np.float32(depth)
        o[:, 1] = (k["y"] - np.float32(cy)) / np.float32(fy) * np.float32(depth)
        o[:, 2] = depth
        return o
    total_matches = 0
    for nb in (1, 2, 3):       # one batch at a time: the last matched batch is then batch nb - 1 of the stream
        r = drv.run(1)
        st = int(r["last_batch"])
        assert st == nb - 1 and r["keypoints"] == int(cnt[st * B:(st + 1) * B].sum()) and r["extract_launches"] > 0
        bk, bd, bc = bufs[st % len(bufs)]
        mp4 = drv.last_matches()
        nm_oracle = 0
        for i in range(B):
            f = st * B + i
            n = int(bc[i])
            assert n == cnt[f]
            assert np.array_equal(bk.numpy()[i, :n].reshape(-1).view(fe.KP_DTYPE), kps[f][:n])
            assert np.array_equal(bd.numpy()[i, :n], desc[f][:n])
            # pair i of a batch: Current = frame f, Last = frame f - 1; the FIRST batch of a run has no predecessor and matches its
            # first frame against its own last frame (a scene cut), later runs continue the stream
            fl = f - 1 if i > 0 else (st * B + B - 1)
            oc = O.OracleFrame(kps[f][:cnt[f]], desc[f][:cnt[f]], w, h)
            ol = O.OracleFrame(kps[fl][:cnt[fl]], desc[fl][:cnt[fl]], w, h)
            n_o, mp_o = O.search_by_projection_ff(oc, ol, np.ones(ol.n, np.uint8), np.zeros(ol.n, np.uint8), world(kps[fl][:cnt[fl]]),
                                                  Tcws[f].reshape(3, 4), fx, fy, cx, cy, th, True)
            assert np.array_equal(mp4[i][:oc.n], mp_o), (st, i)
            nm_oracle += n_o
        assert r["matches"] == nm_oracle
        total_matches += nm_oracle
    assert total_matches > 500
    # two batches in one run: batch 1 of that run takes the last frame of batch 0 as the Last frame of its first pair
    r = drv.run(2)
    st = int(r["last_batch"])
    assert st == 4 and st % NB == 1
    mp4 = drv.last_matches()
    f = (st % NB) * B
    oc = O.OracleFrame(kps[f][:cnt[f]], desc[f][:cnt[f]], w, h)
    ol = O.OracleFrame(kps[f - 1][:cnt[f - 1]], desc[f - 1][:cnt[f - 1]], w, h)
    n_o, mp_o = O.search_by_projection_ff(oc, ol, np.ones(ol.n, np.uint8), np.zeros(ol.n, np.uint8), world(kps[f - 1][:cnt[f - 1]]),
                                          Tcws[f].reshape(3, 4), fx, fy, cx, cy, th, True)
    assert np.array_equal(mp4[0][:oc.n], mp_o) and n_o > 50
    drv.close()
