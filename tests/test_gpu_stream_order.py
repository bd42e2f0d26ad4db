"""Calls on one extractor, matcher or vocabulary handle enqueued on different caller streams, with no host synchronisation
between them: each call's stream waits for the handle's previous call, so the handle's work buffers (the extractor's plan,
level-0 descriptor and tensor map, the matcher's candidate scratch and error flags) serve one call at a time, and the
host-side readers (sync, stage_times, debug_level) see the most recent call whichever stream it ran on.

Every case puts a bounded spin (torch.cuda._sleep, about 50 ms on an H100) on stream A in front of the handle's first call,
enqueues the rest at once and synchronises once at the end.  Every output is compared bit for bit with the oracle.  The
ordering tests check the wait itself: an event recorded on B right after B's call must not complete before A's spin does.
The vocabulary's device entries only read its node table; its cases are a control.

CUDA loads a kernel at its first launch in a process, and that load can wait for the work already on the device: a first
launch behind the spin would be ordered by the load, not by the handle.  So every kernel these cases launch behind a spin
has been launched before, without one (the `loaded` fixture, or a first round of the case itself).
"""
import numpy as np
import pytest

import oracle as O
import orb_slam_b200 as fe
from orb_slam_b200 import bow as B
from orb_slam_b200 import matching as M
from orb_slam_b200.synth import noisy_copies, random_descriptors, random_vocabulary, shifted_frame, textured_frame

import normal_depth_scenes as NDS
from test_gpu_bow_match import _pack_fvs
from test_gpu_normal_depth import _kps, _prefill, _same3, _seeded_store, oracle_of_store

pytestmark = pytest.mark.gpu

SPIN = 100_000_000          # torch.cuda._sleep cycles: one bounded spin of roughly 50 ms on an H100
W, H, NF = 640, 480, 1000
FX = FY = 500.0
CX, CY, DEPTH = W / 2.0, H / 2.0, 4.0


def _torch():
    import torch
    return torch, torch.device("cuda", 0)


def _t(a):
    torch, dev = _torch()
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


@pytest.fixture
def streams(gpu_required):
    """Eight fresh streams; the device is idle when the test starts."""
    torch, dev = _torch()
    ss = [torch.cuda.Stream(device=dev) for _ in range(8)]
    torch.cuda.synchronize()
    return ss


def _spin(s):
    torch, _ = _torch()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SPIN)


def _spin_ms():
    """How long one spin takes on this device, alone on a stream."""
    torch, dev = _torch()
    s = torch.cuda.Stream(device=dev)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(s)
    _spin(s)
    b.record(s)
    b.synchronize()
    return a.elapsed_time(b)


# ---- extractor --------------------------------------------------------------------------------------------------------------------
def _frames(seeds, w=W, h=H):
    return np.stack([textured_frame(w, h, seed=s) for s in seeds])


def _oracle(img):
    rc, k, d, _ = O.extract(O.make_params(NF, 1.2, 8, 1, 20), img)
    assert rc == 0
    return k, d


def _same_kp(gk, gd, ok, od, tag):
    assert len(gk) == len(ok), (tag, len(gk), len(ok))
    for name in ("x", "y", "size", "response", "octave", "class_id"):
        assert np.array_equal(gk[name], ok[name]), (tag, name)
    assert np.array_equal(gk["angle"].view(np.uint32), ok["angle"].view(np.uint32)), tag
    assert np.array_equal(gd, od), tag


class DeviceExtract:
    """One orbfe_extract_batch_device call on `frames` (level 0 read in place, stride = width) into its own outputs."""

    def __init__(self, ex, frames, stream):
        torch, dev = _torch()
        self.frames = frames
        self.B, h, w = frames.shape
        self.cap = int(ex.tables()[2].sum())
        self.d_in = _t(frames)
        self.d_kps = torch.zeros((self.B, self.cap, 28), dtype=torch.uint8, device=dev)
        self.d_desc = torch.zeros((self.B, self.cap, 32), dtype=torch.uint8, device=dev)
        self.d_cnt = torch.full((self.B,), -1, dtype=torch.int32, device=dev)
        self.args = (ex, w, h, stream)

    def enqueue(self):
        ex, w, h, stream = self.args
        ex.extract_batch_device(self.d_in.data_ptr(), w, h, w, w * h, self.B, self.d_kps.data_ptr(), self.d_desc.data_ptr(),
                                self.d_cnt.data_ptr(), stream.cuda_stream)
        return self

    def check(self, tag):
        k = self.d_kps.cpu().numpy().view(fe.KP_DTYPE).reshape(self.B, self.cap)
        d, c = self.d_desc.cpu().numpy(), self.d_cnt.cpu().numpy()
        for f in range(self.B):
            _same_kp(k[f, :c[f]], d[f, :c[f]], *_oracle(self.frames[f]), (tag, f))


def test_frames_written_behind_a_spin_are_the_ones_extracted(streams):
    """The input is overwritten on A behind a spin, then extracted in place on A: the keypoints are those of the new frames."""
    torch, _ = _torch()
    A = streams[0]
    ex = fe.ORBextractor(NF, 1.2, 8)
    try:
        call = DeviceExtract(ex, _frames([1, 2]), A)
        final = _frames([3, 4])
        d_final = _t(final)
        torch.cuda.synchronize()
        _spin(A)
        with torch.cuda.stream(A):
            call.d_in.copy_(d_final)
        call.frames = final
        call.enqueue()
        torch.cuda.synchronize()
        call.check("overwritten")
    finally:
        ex.close()


@pytest.mark.parametrize("ingest", ["in_place", "copy", "one_of_each"])
def test_two_device_calls_on_two_streams(streams, monkeypatch, ingest):
    """A call on A behind a spin, then at once a call with other frames on B: B's call does not rewrite level 0, the tensor
    map or the work buffers under A's."""
    torch, _ = _torch()
    A, Bs = streams[:2]
    ex = fe.ORBextractor(NF, 1.2, 8)
    try:
        first, second = DeviceExtract(ex, _frames([11, 12]), A), DeviceExtract(ex, _frames([13, 14]), Bs)
        ex.extract_batch(first.frames)                  # the plan exists: no call below rebuilds it
        torch.cuda.synchronize()
        if ingest == "copy":
            monkeypatch.setenv("ORBFE_INGEST_COPY", "1")
        _spin(A)
        first.enqueue()
        if ingest == "one_of_each":
            monkeypatch.setenv("ORBFE_INGEST_COPY", "1")
        second.enqueue()
        torch.cuda.synchronize()
        first.check("first")
        second.check("second")
    finally:
        ex.close()


@pytest.mark.parametrize("batch_mode", [0, 1])
def test_host_extracts_after_a_pending_device_call(streams, batch_mode):
    """A device call of 8 frames on A behind a spin, then orbfe_extract and an 8-frame orbfe_extract_batch (four upload chunks
    on the copy stream): the host calls wait for the device call, whose outputs stay its own."""
    torch, _ = _torch()
    A = streams[0]
    ex = fe.ORBextractor(NF, 1.2, 8)
    ex.set_batch_mode(batch_mode)
    try:
        call = DeviceExtract(ex, _frames(range(20, 28)), A)
        ex.extract_batch(call.frames)                   # the plan for 8 frames at this geometry
        single, batch = textured_frame(W, H, seed=30), _frames(range(31, 39))
        torch.cuda.synchronize()
        _spin(A)
        call.enqueue()
        gk, gd = ex(single)
        kps, desc, cnt = ex.extract_batch(batch)
        torch.cuda.synchronize()
        _same_kp(gk, gd, *_oracle(single), "orbfe_extract")
        for f in range(len(batch)):
            _same_kp(kps[f, :cnt[f]], desc[f, :cnt[f]], *_oracle(batch[f]), ("orbfe_extract_batch", f))
        call.check("device")
    finally:
        ex.close()


def test_debug_level_reads_the_pending_call(streams):
    """A device call on A behind a spin, then debug_level for every level of both frames: the pyramid and the blurred levels
    of that call."""
    A = streams[0]
    ex = fe.ORBextractor(NF, 1.2, 8)
    try:
        frames = _frames([41, 42])
        ex.extract_batch(_frames([43, 44]))         # the levels a read that did not wait would return
        _spin(A)
        DeviceExtract(ex, frames, A).enqueue()
        got = [[(ex.debug_level(f, l, False), ex.debug_level(f, l, True)) for l in range(8)] for f in range(2)]
        for f in range(2):
            rc, _, _, dump = O.extract(O.make_params(NF, 1.2, 8, 1, 20), frames[f], want_dump=True)
            assert rc == 0
            for l in range(8):
                assert np.array_equal(got[f][l][0], dump["levels"][l][O.EDGE:-O.EDGE, O.EDGE:-O.EDGE]), (f, l)
                if dump["n_level_kp"][l] > 0:     # the oracle smooths only the levels that have keypoints
                    assert np.array_equal(got[f][l][1], dump["blurred"][l][O.EDGE:-O.EDGE, O.EDGE:-O.EDGE]), (f, l)
    finally:
        ex.close()


def test_geometry_change_on_another_stream(streams):
    """A 640x480 call on A behind a spin, then an 800x608 call on B, which rebuilds the plan: the rebuild waits for A's call."""
    torch, _ = _torch()
    A, Bs = streams[:2]
    ex = fe.ORBextractor(NF, 1.2, 8)
    try:
        first, second = DeviceExtract(ex, _frames([51, 52]), A), DeviceExtract(ex, _frames([53, 54], 800, 608), Bs)
        ex.extract_batch(first.frames)
        torch.cuda.synchronize()
        _spin(A)
        first.enqueue()
        second.enqueue()
        torch.cuda.synchronize()
        first.check("640x480")
        second.check("800x608")
    finally:
        ex.close()


def test_eight_calls_round_robin_on_eight_streams(streams):
    torch, _ = _torch()
    ex = fe.ORBextractor(NF, 1.2, 8)
    try:
        calls = [DeviceExtract(ex, _frames([60 + i]), s) for i, s in enumerate(streams)]
        ex.extract_batch(calls[0].frames)
        torch.cuda.synchronize()
        _spin(streams[0])
        for c in calls:
            c.enqueue()
        torch.cuda.synchronize()
        for i, c in enumerate(calls):
            c.check(i)
    finally:
        ex.close()


STAGES = ["ingest", "pyramid", "fast_nms", "cell_quota", "cell_select", "level_select", "describe"]


def test_stage_times_of_calls_on_two_streams(streams):
    """Profiling on, a call on A behind a spin and one on B: stage_times returns the intervals of both calls at once."""
    torch, _ = _torch()
    A, Bs = streams[:2]
    ex = fe.ORBextractor(NF, 1.2, 8)
    try:
        first, second = DeviceExtract(ex, _frames([71]), A), DeviceExtract(ex, _frames([72]), Bs)
        ex.extract_batch(first.frames)
        torch.cuda.synchronize()
        ex.set_profiling(True)
        _spin(A)
        first.enqueue()
        second.enqueue()
        st = ex.stage_times()
        assert [n for n, _ in st] == STAGES + STAGES, st
        assert all(np.isfinite(ms) and ms >= 0 for _, ms in st), st
        torch.cuda.synchronize()
        first.check("A")
        second.check("B")
    finally:
        ex.close()


def test_extractor_call_on_b_waits_for_the_call_on_a(streams):
    torch, _ = _torch()
    A, Bs = streams[:2]
    spin = _spin_ms()
    ex = fe.ORBextractor(NF, 1.2, 8)
    try:
        first, second = DeviceExtract(ex, _frames([81]), A), DeviceExtract(ex, _frames([82]), Bs)
        ex.extract_batch(first.frames)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(A)
        _spin(A)
        first.enqueue()
        second.enqueue()
        e1.record(Bs)
        assert not e1.query()
        e1.synchronize()
        assert e0.elapsed_time(e1) >= 0.8 * spin, (e0.elapsed_time(e1), spin)
        torch.cuda.synchronize()
        first.check("A")
        second.check("B")
    finally:
        ex.close()


# ---- matcher: the fused windowed kernel ------------------------------------------------------------------------------------------------
def _features(n_frames):
    """Extracted features of a synthetic stream (frame i is frame i-1 shifted by a few pixels), as in test_gpu_matchers."""
    ex = fe.ORBextractor(NF, 1.2, 8)
    frames, shifts = [textured_frame(W, H, seed=21)], [(0, 0)]
    rng = np.random.default_rng(1)
    for i in range(1, n_frames):
        dx, dy = int(rng.integers(-5, 6)), int(rng.integers(-4, 5))
        frames.append(shifted_frame(frames[-1], dx, dy, seed=i))
        shifts.append((dx, dy))
    feats = [ex(f) for f in frames]
    ex.close()
    return feats, shifts


def _store(feats, trim):
    """The frame store (cap NF), frame f keeping all but trim * f features."""
    nfr = len(feats)
    kps, desc, counts = np.zeros((nfr, NF), fe.KP_DTYPE), np.zeros((nfr, NF, 32), np.uint8), np.zeros(nfr, np.int32)
    for f, (k, d) in enumerate(feats):
        n = len(k) - trim * f
        kps[f, :n], desc[f, :n], counts[f] = k[:n], d[:n], n
    return kps, desc, counts


def _oframe(kps, desc, counts, f):
    return O.OracleFrame(kps[f, :counts[f]], desc[f, :counts[f]], W, H)


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
def scene(gpu_required):
    feats, shifts = _features(5)
    return feats, shifts, _store(feats, 29)


@pytest.fixture(scope="module", autouse=True)
def loaded(gpu_required, scene):
    """Every extractor and fused-matcher kernel of this file launched once, with nothing else on the device."""
    torch, dev = _torch()
    s = torch.cuda.Stream(device=dev)
    ex = fe.ORBextractor(NF, 1.2, 8)
    m = fe.ORBmatcher(0.9, True)
    try:
        frames = _frames([1, 2])
        ex.extract_batch(frames)
        call = DeviceExtract(ex, frames, s).enqueue()
        with torch.cuda.stream(s):
            call.d_in.copy_(call.d_in.flip(0))
        ex.debug_level(0, 0, True)
        InitCall(scene[2], [(0, 1)]).enqueue(m, s)
        SbpCall(scene, [(1, 0)], 1).enqueue(m, s)
        GuidedCall(scene, [(1, 0)], 0, 60, 1).enqueue(m, s)
        (k1, d1), (k2, d2) = scene[0][:2]
        M.window_search(m, M.FrameView(k1, d1, W, H), M.FrameView(k2, d2, W, H), np.ones(len(k1), np.uint8), 50)
        torch.cuda.synchronize()
        m.sync()
    finally:
        m.close()
        ex.close()


class InitCall:
    """orbfe_search_for_initialization_device over `pairs` of the store, into its own outputs."""

    def __init__(self, store, pairs):
        torch, dev = _torch()
        kps, desc, counts = store
        self.store, self.pairs = store, pairs
        self.d = [_t(kps.view(np.uint8).reshape(len(counts), NF, 28)), _t(desc), _t(counts)]
        self.prev = np.zeros((len(pairs), NF, 2), np.float32)
        for j, (a, _) in enumerate(pairs):
            self.prev[j, :, 0], self.prev[j, :, 1] = kps[a]["x"], kps[a]["y"]
        self.d_f1, self.d_f2 = _t(np.array([p[0] for p in pairs], np.int32)), _t(np.array([p[1] for p in pairs], np.int32))
        self.d_prev = _t(self.prev)
        self.d_m12 = torch.full((len(pairs), NF), -7, dtype=torch.int32, device=dev)
        self.d_nm = torch.full((len(pairs),), -7, dtype=torch.int32, device=dev)

    def enqueue(self, m, stream):
        M.search_for_initialization_device(m, len(self.pairs), *[x.data_ptr() for x in self.d], NF, self.d_f1.data_ptr(),
                                           self.d_f2.data_ptr(), self.d_prev.data_ptr(), W, H, 100, self.d_m12.data_ptr(),
                                           self.d_nm.data_ptr(), stream.cuda_stream)

    def check(self, m, tag):
        kps, desc, counts = self.store
        m12, nm, pv = self.d_m12.cpu().numpy(), self.d_nm.cpu().numpy(), self.d_prev.cpu().numpy()
        for j, (a, b) in enumerate(self.pairs):
            n_o, m_o, p_o = O.search_for_initialization(_oframe(kps, desc, counts, a), _oframe(kps, desc, counts, b),
                                                        self.prev[j, :counts[a]], 100, nnratio=float(m.mfNNratio),
                                                        check_orientation=m.mbCheckOrientation)
            assert nm[j] == n_o, (tag, j, nm[j], n_o)
            assert np.array_equal(m12[j, :counts[a]], m_o), (tag, j)
            assert np.array_equal(pv[j, :counts[a]], p_o), (tag, j)
        return int(nm.sum())


def test_search_for_initialization_on_two_streams(streams, scene):
    """Both launches read and write the global candidate scratch: B's waits for A's."""
    torch, _ = _torch()
    A, Bs = streams[:2]
    first, second = InitCall(scene[2], [(0, 1), (2, 3), (1, 2)]), InitCall(scene[2], [(1, 0), (3, 2)])
    m = fe.ORBmatcher(0.9, True)
    try:
        torch.cuda.synchronize()
        _spin(A)
        first.enqueue(m, A)
        second.enqueue(m, Bs)
        torch.cuda.synchronize()
        m.sync()
        assert first.check(m, "A") > 50 and second.check(m, "B") > 50
    finally:
        m.close()


class SbpCall:
    """orbfe_search_by_projection_device over (Current, Last) `pairs` of the store, Last's map points at DEPTH."""

    def __init__(self, scene, pairs, seed):
        torch, dev = _torch()
        feats, shifts, (kps, desc, counts) = scene
        rng = np.random.default_rng(seed)
        nfr = len(counts)
        self.kps, self.desc, self.counts, self.pairs = kps, desc, counts, pairs
        self.world = np.stack([_world(kps[f]) for f in range(nfr)])
        self.flags = (rng.random((nfr, NF)) < 0.92).astype(np.uint8)
        self.T = np.stack([_tcw(*shifts[c]) if c == l + 1 else _tcw(0, 0) for c, l in pairs]).astype(np.float32)
        self.pre = np.full((len(pairs), NF), -1, np.int32)
        self.pre[rng.random((len(pairs), NF)) < 0.02] = 7
        self.d = [_t(kps.view(np.uint8).reshape(nfr, NF, 28)), _t(desc), _t(counts), _t(np.array([p[0] for p in pairs], np.int32)),
                  _t(np.array([p[1] for p in pairs], np.int32)), _t(self.world), _t(self.flags), _t(self.T.reshape(len(pairs), 12))]
        self.d_mp, self.d_nm = _t(self.pre), torch.full((len(pairs),), -7, dtype=torch.int32, device=dev)

    def enqueue(self, m, stream):
        M.search_by_projection_device(m, len(self.pairs), *[x.data_ptr() for x in self.d[:3]], NF, *[x.data_ptr() for x in self.d[3:]],
                                      W, H, 1.2, 8, FX, FY, CX, CY, 15.0, self.d_mp.data_ptr(), self.d_nm.data_ptr(), stream.cuda_stream)

    def check(self, m, tag):
        mp, nm = self.d_mp.cpu().numpy(), self.d_nm.cpu().numpy()
        c_ = self.counts
        for j, (c, l) in enumerate(self.pairs):
            n_o, mp_o = O.search_by_projection_ff(_oframe(self.kps, self.desc, c_, c), _oframe(self.kps, self.desc, c_, l),
                                                  self.flags[l, :c_[l]], np.zeros(c_[l], np.uint8), self.world[l, :c_[l]], self.T[j],
                                                  FX, FY, CX, CY, 15.0, m.mbCheckOrientation, cur_mp=self.pre[j, :c_[c]])
            assert nm[j] == n_o, (tag, j, nm[j], n_o)
            assert np.array_equal(mp[j, :c_[c]], mp_o), (tag, j)
        return int(nm.sum())


@pytest.mark.parametrize("force_scratch", [False, True])
def test_search_by_projection_on_two_streams(streams, scene, monkeypatch, force_scratch):
    torch, _ = _torch()
    if force_scratch:
        monkeypatch.setenv("ORBFE_SBP_FORCE_SCRATCH", "1")
    A, Bs = streams[:2]
    first, second = SbpCall(scene, [(1, 0), (2, 1), (3, 2)], 5), SbpCall(scene, [(4, 3), (2, 2), (4, 0)], 6)
    m = fe.ORBmatcher(0.9, True)
    try:
        torch.cuda.synchronize()
        _spin(A)
        first.enqueue(m, A)
        second.enqueue(m, Bs)
        torch.cuda.synchronize()
        m.sync()
        assert first.check(m, "A") > 200 and second.check(m, "B") > 200
    finally:
        m.close()


class GuidedCall:
    """orbfe_guided_search_device: job j searches frame jobs[j][0] with the features of frame jobs[j][1], moved by the shift."""

    def __init__(self, scene, jobs, rule, th, seed):
        torch, dev = _torch()
        feats, shifts, (kps, desc, counts) = scene
        rng = np.random.default_rng(seed)
        q = {k: [] for k in ("u", "v", "r", "lo", "hi", "d", "a")}
        qbase, qcnt = [], []
        for tgt, src in jobs:
            k, d = kps[src, :counts[src]], desc[src, :counts[src]]
            keep = rng.random(len(k)) < 0.8
            k, d = k[keep], d[keep]
            dx = sum(s[0] for s in shifts[min(src, tgt) + 1:max(src, tgt) + 1]) * (1 if tgt > src else -1)
            dy = sum(s[1] for s in shifts[min(src, tgt) + 1:max(src, tgt) + 1]) * (1 if tgt > src else -1)
            qbase.append(sum(qcnt))
            qcnt.append(len(k))
            q["u"].append(k["x"] + np.float32(dx) + rng.normal(0, 1.0, len(k)).astype(np.float32))
            q["v"].append(k["y"] + np.float32(dy) + rng.normal(0, 1.0, len(k)).astype(np.float32))
            q["r"].append((np.float32(7.0) * np.float32(1.2) ** k["octave"]).astype(np.float32))
            q["lo"].append((k["octave"] - 1).astype(np.int32))
            q["hi"].append((k["octave"] + 1).astype(np.int32))
            q["d"].append(d)
            q["a"].append(k["angle"])
        types = dict(u=np.float32, v=np.float32, r=np.float32, lo=np.int32, hi=np.int32, d=np.uint8, a=np.float32)
        self.q = {k: np.ascontiguousarray(np.concatenate(v).astype(types[k])) for k, v in q.items()}
        self.kps, self.desc, self.counts, self.jobs, self.rule, self.th = kps, desc, counts, jobs, rule, th
        self.qbase, self.qcnt = qbase, qcnt
        self.pre = np.full((len(jobs), NF), -1, np.int32)
        self.pre[rng.random((len(jobs), NF)) < 0.03] = 4
        self.d = [_t(kps.view(np.uint8).reshape(len(counts), NF, 28)), _t(desc), _t(counts), _t(np.array([j[0] for j in jobs], np.int32))]
        self.d_q = [_t(self.q[k]) for k in ("u", "v", "r", "lo", "hi", "d", "a")]
        self.d_qb, self.d_qc = _t(np.array(qbase, np.int32)), _t(np.array(qcnt, np.int32))
        self.d_so, self.d_nm = _t(self.pre), torch.full((len(jobs),), -7, dtype=torch.int32, device=dev)

    def enqueue(self, m, stream):
        M.guided_search_device(m, len(self.jobs), *[x.data_ptr() for x in self.d[:3]], NF, self.d[3].data_ptr(),
                               *[x.data_ptr() for x in self.d_q], self.d_qb.data_ptr(), self.d_qc.data_ptr(), max(self.qcnt), W, H,
                               self.rule, self.th, self.d_so.data_ptr(), self.d_nm.data_ptr(), stream.cuda_stream)

    def check(self, m, tag):
        so, nm = self.d_so.cpu().numpy(), self.d_nm.cpu().numpy()
        for j, (tgt, _) in enumerate(self.jobs):
            sl = slice(self.qbase[j], self.qbase[j] + self.qcnt[j])
            n_o, so_o = O.guided_search(_oframe(self.kps, self.desc, self.counts, tgt), *[self.q[k][sl] for k in ("u", "v", "r", "lo", "hi", "d", "a")],
                                        self.rule, float(m.mfNNratio), self.th, 1 if m.mbCheckOrientation else 0,
                                        slot_owner=self.pre[j, :self.counts[tgt]])
            assert nm[j] == n_o, (tag, j, nm[j], n_o)
            assert np.array_equal(so[j, :self.counts[tgt]], so_o), (tag, j)
        return int(nm.sum())


@pytest.mark.parametrize("force_scratch", [False, True])
def test_guided_search_on_two_streams(streams, scene, monkeypatch, force_scratch):
    torch, _ = _torch()
    if force_scratch:
        monkeypatch.setenv("ORBFE_SBP_FORCE_SCRATCH", "1")
    A, Bs = streams[:2]
    first, second = GuidedCall(scene, [(1, 0), (2, 1), (3, 2)], 1, 0, 7), GuidedCall(scene, [(0, 3), (2, 2), (4, 3)], 0, 60, 8)
    m = fe.ORBmatcher(0.8, True)
    try:
        torch.cuda.synchronize()
        _spin(A)
        first.enqueue(m, A)
        second.enqueue(m, Bs)
        torch.cuda.synchronize()
        m.sync()
        assert first.check(m, "A") > 100 and second.check(m, "B") > 100
    finally:
        m.close()


def test_host_window_search_after_a_pending_device_call(streams, scene):
    """A device call on A behind a spin, then a host-array window search with whole-image windows on the matcher's own stream:
    every candidate list holds every feature, so the call runs again with a grown scratch, which waits for A's call."""
    torch, _ = _torch()
    A = streams[0]
    feats = scene[0]
    (k1, d1), (k2, d2) = feats[0], feats[1]
    has = (np.random.default_rng(0).random(len(k1)) < 0.8).astype(np.uint8)
    first = SbpCall(scene, [(1, 0)], 9)
    m = fe.ORBmatcher(0.9, True)
    try:
        torch.cuda.synchronize()
        _spin(A)
        first.enqueue(m, A)
        n, m21 = M.window_search(m, M.FrameView(k1, d1, W, H), M.FrameView(k2, d2, W, H), has, 1000)
        torch.cuda.synchronize()
        m.sync()
        n_o, m21_o = O.window_search(O.OracleFrame(k1, d1, W, H), O.OracleFrame(k2, d2, W, H), has, 1000, nnratio=0.9,
                                     check_orientation=True)
        assert n == n_o and np.array_equal(m21, m21_o)
        assert n > 20
        assert first.check(m, "device") > 50
    finally:
        m.close()


def test_larger_call_on_b_grows_the_scratch_after_a(streams, scene, monkeypatch):
    """A one-pair call on A behind a spin, then five pairs on B: B's call needs a larger scratch, which is freed only after A's
    call has ended."""
    torch, _ = _torch()
    monkeypatch.setenv("ORBFE_SBP_FORCE_SCRATCH", "1")
    A, Bs = streams[:2]
    first, second = SbpCall(scene, [(1, 0)], 10), SbpCall(scene, [(1, 0), (2, 1), (3, 2), (4, 3), (4, 0)], 11)
    m = fe.ORBmatcher(0.9, False)
    try:
        torch.cuda.synchronize()
        _spin(A)
        first.enqueue(m, A)
        second.enqueue(m, Bs)
        torch.cuda.synchronize()
        m.sync()
        assert first.check(m, "A") > 50 and second.check(m, "B") > 200
    finally:
        m.close()


# ---- matcher: error flags ------------------------------------------------------------------------------------------------------------
def test_sync_reports_the_pending_malformed_call(streams):
    """A normal_and_depth_device call with a reference slot beyond the store, on A behind a spin; m.sync() at once raises
    ORBFE_ERR_ARG naming that entry, and the next sync is clean."""
    torch, _ = _torch()
    A = streams[0]
    octs, counts, centers, gp, obs, ref, world = _seeded_store(5, nframes=12, cap=512, npoints=400)
    nf, cap = len(counts), 512
    ref = ref.copy()
    ref[3] = nf * cap
    n = len(gp) - 1
    d_kps, d_cnt, d_c, d_gp, d_obs, d_ref, d_w = (_t(x) for x in (_kps(octs).view(np.uint8), counts, centers, gp, obs, ref, world))
    d_out = [_t(x) for x in _prefill(n)]
    m = fe.ORBmatcher(0.6, True)
    try:
        for spun in (False, True):
            torch.cuda.synchronize()
            if spun:
                _spin(A)
            B.normal_and_depth_device(m, n, d_kps.data_ptr(), d_cnt.data_ptr(), nf, cap, d_c.data_ptr(), d_gp.data_ptr(), d_obs.data_ptr(),
                                      len(obs), d_w.data_ptr(), d_ref.data_ptr(), 1.2, NDS.scale_table(1.2, 8),
                                      *[x.data_ptr() for x in d_out], A.cuda_stream)
            with pytest.raises(fe.OrbfeError) as e:
                m.sync()
            assert e.value.code == fe.ORBFE_ERR_ARG and "orbfe_normal_and_depth_device" in str(e.value), spun
            m.sync()
    finally:
        m.close()


# ---- matcher: BoW, map-point and stateless entries -----------------------------------------------------------------------------------
def _bow_pair(seed, n1=1500, n2=1400):
    """Two frames of one synthetic scene for SearchByBoW (frame 1 sees noisy copies of a subset of frame 0's features)."""
    rng = np.random.default_rng(seed)
    d1 = random_descriptors(n1, seed)
    perm = rng.permutation(n1)[:n2]
    d2 = noisy_copies(d1[perm], 0.05, seed + 1)
    a1 = rng.uniform(0, 360, n1).astype(np.float32)
    a2 = ((a1[perm] + rng.normal(7, 4, n2)) % 360).astype(np.float32)
    node1 = (d1[:, 0].astype(np.int32) >> 3) * 3 + 11
    node2 = (d2[:, 0].astype(np.int32) >> 3) * 3 + 11
    valid = [(rng.random(n1) < 0.8).astype(np.uint8), (rng.random(n2) < 0.9).astype(np.uint8)]
    return [d1, d2], [a1, a2], [M.feature_vector(node1), M.feature_vector(node2)], valid


def test_map_point_bow_and_stateless_entries_alternating(streams, scene):
    """search_by_bow_device, search_for_triangulation_device, distinctive_descriptors_device, normal_and_depth_device,
    knn2_groups_device, hamming_csr_device and undistort_keypoints_device on one matcher, alternating between A (first
    behind a spin) and B, then one synchronisation: every output equals its oracle."""
    torch, dev = _torch()
    A, Bs = streams[:2]
    S = [A, Bs]
    m = fe.ORBmatcher(0.75, True)
    checks = []
    # SearchByBoW, one job (KeyFrame vs KeyFrame)
    desc2, ang2, fv2, valid2 = _bow_pair(21)
    cap = 1500
    kb = np.zeros((2, cap), fe.KP_DTYPE)
    db = np.zeros((2, cap, 32), np.uint8)
    vb = np.zeros((2, cap), np.uint8)
    for f in range(2):
        n = len(desc2[f])
        kb[f, :n]["angle"], db[f, :n], vb[f, :n] = ang2[f], desc2[f], valid2[f]
    fvb = [_t(x) for x in _pack_fvs(fv2, cap)]
    d_bow = [_t(kb.view(np.uint8).reshape(2, cap, 28)), _t(db), _t(np.array([len(x) for x in desc2], np.int32))]
    d_bv, d_i1, d_i2 = _t(vb), _t(np.array([0], np.int32)), _t(np.array([1], np.int32))
    d_bout, d_bnm = torch.full((1, cap), -9, dtype=torch.int32, device=dev), torch.full((1,), -9, dtype=torch.int32, device=dev)

    def bow(s):
        M.search_by_bow_device(m, 1, 1, *[x.data_ptr() for x in d_bow], cap, *[x.data_ptr() for x in fvb], d_bv.data_ptr(),
                               d_i1.data_ptr(), d_i2.data_ptr(), d_bout.data_ptr(), d_bnm.data_ptr(), s.cuda_stream)

    def bow_check():
        n_o, out_o = O.search_by_bow(1, desc2[0], valid2[0], ang2[0], fv2[0], desc2[1], valid2[1], ang2[1], fv2[1], nnratio=0.75,
                                     check_orientation=True)
        assert d_bnm.cpu().numpy()[0] == n_o and n_o > 300
        assert np.array_equal(d_bout.cpu().numpy()[0, :len(desc2[0])], out_o)

    # SearchForTriangulation, one job between the first two frames of the stream
    feats, shifts, _ = scene
    (k1, d1), (k2, d2) = feats[0], feats[1]
    rng = np.random.default_rng(31)
    tri_has = [(rng.random(len(k1)) < 0.4).astype(np.uint8), (rng.random(len(k2)) < 0.4).astype(np.uint8)]
    tri_fv = [M.feature_vector((d[:, 3].astype(np.int32) >> 4) * 7 + 2) for d in (d1, d2)]
    F12 = np.array([[0, 0, 0], [0, 0, -1], [0, 1, float(-shifts[1][1])]], np.float32)
    sigma2 = (np.float32(1.2) ** np.arange(8, dtype=np.float32)) ** 2
    kt, dt, ht = np.zeros((2, NF), fe.KP_DTYPE), np.zeros((2, NF, 32), np.uint8), np.zeros((2, NF), np.uint8)
    for f, (k, d) in enumerate(((k1, d1), (k2, d2))):
        kt[f, :len(k)], dt[f, :len(k)], ht[f, :len(k)] = k, d, tri_has[f]
    d_tri = [_t(kt.view(np.uint8).reshape(2, NF, 28)), _t(dt), _t(np.array([len(k1), len(k2)], np.int32))]
    fvt = [_t(x) for x in _pack_fvs(tri_fv, NF)]
    d_th, d_F = _t(ht), _t(F12.reshape(1, 9))
    d_tout, d_tnm = torch.full((1, NF), -9, dtype=torch.int32, device=dev), torch.full((1,), -9, dtype=torch.int32, device=dev)

    def tri(s):
        M.search_for_triangulation_device(m, 1, *[x.data_ptr() for x in d_tri], NF, *[x.data_ptr() for x in fvt], d_th.data_ptr(),
                                          d_i1.data_ptr(), d_i2.data_ptr(), d_F.data_ptr(), sigma2, d_tout.data_ptr(), d_tnm.data_ptr(),
                                          s.cuda_stream)

    def tri_check():
        n_o, m12_o = O.search_for_triangulation(k1, d1, tri_has[0], tri_fv[0], k2, d2, tri_has[1], tri_fv[1], F12, sigma2,
                                                check_orientation=True)
        assert d_tnm.cpu().numpy()[0] == n_o and n_o > 20
        assert np.array_equal(d_tout.cpu().numpy()[0, :len(k1)], m12_o)

    # ComputeDistinctiveDescriptors and UpdateNormalAndDepth on one frame store
    octs, counts, centers, gp, obs, ref, world = _seeded_store(13, nframes=60, cap=1024, npoints=2000)
    nfs, scap = len(counts), 1024
    sizes = np.minimum(np.diff(gp), 150)
    obs = np.concatenate([obs[gp[g]:gp[g] + sizes[g]] for g in range(len(sizes))]).astype(np.int32)
    gp = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    sdesc = np.random.default_rng(13).integers(0, 256, (nfs * scap, 32), dtype=np.uint8)
    npts = len(gp) - 1
    d_sd, d_sk, d_sc, d_cc, d_gp, d_obs, d_ref, d_w = (_t(x) for x in (sdesc, _kps(octs).view(np.uint8), counts, centers, gp, obs, ref, world))
    d_best = torch.full((npts,), -9, dtype=torch.int32, device=dev)
    d_mpd = torch.zeros((npts, 32), dtype=torch.uint8, device=dev)
    d_nd = [_t(x) for x in _prefill(npts)]
    sfs = NDS.scale_table(1.2, 8)

    def distinctive(s):
        B.distinctive_descriptors_device(m, npts, d_sd.data_ptr(), d_sc.data_ptr(), nfs, scap, d_gp.data_ptr(), d_obs.data_ptr(), len(obs),
                                         d_best.data_ptr(), d_mpd.data_ptr(), s.cuda_stream)

    def distinctive_check():
        best = O.distinctive_descriptors(sdesc[obs], gp)
        assert np.array_equal(d_best.cpu().numpy(), best)
        assert np.array_equal(d_mpd.cpu().numpy(), sdesc[obs[gp[:-1] + best]])

    def normal_depth(s):
        B.normal_and_depth_device(m, npts, d_sk.data_ptr(), d_sc.data_ptr(), nfs, scap, d_cc.data_ptr(), d_gp.data_ptr(), d_obs.data_ptr(),
                                  len(obs), d_w.data_ptr(), d_ref.data_ptr(), 1.2, sfs, *[x.data_ptr() for x in d_nd], s.cuda_stream)

    def normal_depth_check():
        got = tuple(x.cpu().numpy() for x in d_nd)
        assert _same3(got, oracle_of_store(octs, counts, centers, gp, obs, ref, world, 1.2, sfs))

    # knn2 over groups and Hamming distances of CSR pairs
    q, kdb = random_descriptors(256, 1), random_descriptors(12 * 500, 2)
    d_q, d_kdb = _t(q), _t(kdb)
    d_kb, d_ki, d_ks = (torch.zeros((12, 256), dtype=t, device=dev) for t in (torch.uint16, torch.int32, torch.uint16))

    def knn2(s):
        fe.lib().orbfe_knn2_groups_device(m.handle, d_q.data_ptr(), 256, d_kdb.data_ptr(), 12, 500, d_kb.data_ptr(), d_ki.data_ptr(),
                                          d_ks.data_ptr(), s.cuda_stream)

    def knn2_check():
        for g in range(12):
            bd, bi, sd = O.knn2(q, kdb[g * 500:(g + 1) * 500])
            assert np.array_equal(d_kb[g].cpu().numpy(), bd) and np.array_equal(d_ki[g].cpu().numpy(), bi)
            assert np.array_equal(d_ks[g].cpu().numpy(), np.minimum(sd, 65535))

    row_ptr = np.concatenate([[0], np.cumsum(rng.integers(0, 40, 256))]).astype(np.int32)
    cols = rng.integers(0, len(kdb), int(row_ptr[-1])).astype(np.int32)
    d_rp, d_cols = _t(row_ptr), _t(cols)
    d_ham = torch.zeros(len(cols), dtype=torch.uint16, device=dev)

    def hamming(s):
        fe.lib().orbfe_hamming_csr_device(m.handle, d_q.data_ptr(), d_kdb.data_ptr(), d_rp.data_ptr(), d_cols.data_ptr(), 256, len(cols),
                                          d_ham.data_ptr(), s.cuda_stream)

    def hamming_check():
        rows = np.repeat(np.arange(256), np.diff(row_ptr))
        want = np.unpackbits(np.bitwise_xor(q[rows], kdb[cols]), axis=1).sum(axis=1)
        assert np.array_equal(d_ham.cpu().numpy(), want)

    # Frame::UndistortKeyPoints, out of place
    ku = feats[2][0].copy()
    dist = [0.12, -0.21, 0.001, -0.002, 0.05]
    d_ku, d_kuo = _t(ku.view(np.uint8).reshape(len(ku), 28)), torch.zeros((len(ku), 28), dtype=torch.uint8, device=dev)

    def undistort(s):
        M.undistort_keypoints_device(m, d_ku.data_ptr(), d_kuo.data_ptr(), len(ku), FX, FY, CX, CY, dist, s.cuda_stream)

    def undistort_check():
        got = d_kuo.cpu().numpy().reshape(-1).view(fe.KP_DTYPE)
        assert np.array_equal(got.view(np.uint8), O.undistort_keypoints(ku, FX, FY, CX, CY, dist).view(np.uint8))

    calls = [(bow, bow_check), (tri, tri_check), (distinctive, distinctive_check), (normal_depth, normal_depth_check),
             (knn2, knn2_check), (hamming, hamming_check), (undistort, undistort_check)]
    try:
        for spun in (False, True):     # the calls rewrite their outputs with the same values
            torch.cuda.synchronize()
            if spun:
                _spin(A)
            for i, (call, _) in enumerate(calls):
                call(S[i % 2])
            torch.cuda.synchronize()
            m.sync()
            for _, check in calls:
                check()
    finally:
        m.close()


# ---- ordering itself -------------------------------------------------------------------------------------------------------------------
def test_matcher_call_on_b_waits_for_the_call_on_a(streams):
    """Undistortion on A behind a spin, then on B: an event recorded on B right after B's call completes only after the spin."""
    torch, dev = _torch()
    A, Bs = streams[:2]
    spin = _spin_ms()
    ku = _features(1)[0][0][0]
    dist = [0.12, -0.21, 0.001, -0.002, 0.05]
    d_in = _t(ku.view(np.uint8).reshape(len(ku), 28))
    outs = [torch.zeros((len(ku), 28), dtype=torch.uint8, device=dev) for _ in range(2)]
    m = fe.ORBmatcher(0.9, True)
    try:
        M.undistort_keypoints_device(m, d_in.data_ptr(), outs[0].data_ptr(), len(ku), FX, FY, CX, CY, dist, A.cuda_stream)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(A)
        _spin(A)
        M.undistort_keypoints_device(m, d_in.data_ptr(), outs[0].data_ptr(), len(ku), FX, FY, CX, CY, dist, A.cuda_stream)
        M.undistort_keypoints_device(m, d_in.data_ptr(), outs[1].data_ptr(), len(ku), FX, FY, CX, CY, dist, Bs.cuda_stream)
        e1.record(Bs)
        assert not e1.query()
        e1.synchronize()
        assert e0.elapsed_time(e1) >= 0.8 * spin, (e0.elapsed_time(e1), spin)
        torch.cuda.synchronize()
        want = O.undistort_keypoints(ku, FX, FY, CX, CY, dist).view(np.uint8)
        for o in outs:
            assert np.array_equal(o.cpu().numpy().reshape(-1), want.reshape(-1))
    finally:
        m.close()


# ---- vocabulary (control) --------------------------------------------------------------------------------------------------------------
def test_vocabulary_device_entries_on_two_streams(streams):
    """descend_device, feature_vector_device, bow_vector_device and min_score_device over two streams behind a spin, with a host
    transform on the same vocabulary in between: all equal the oracle and the host transform."""
    torch, dev = _torch()
    A, Bs = streams[:2]
    voc = random_vocabulary(10, 4, seed=14)
    F, cap, levelsup = 4, 600, 2
    desc = np.stack([random_descriptors(cap, 90 + f) for f in range(F)])
    counts = np.array([600, 517, 0, 333], np.int32)
    v = B.Vocabulary(voc)
    try:
        d_desc, d_cnt = _t(desc), _t(counts)
        d_leaf, d_node = (torch.full((F * cap,), -7, dtype=torch.int32, device=dev) for _ in range(2))
        d_fv = [torch.full(s, -7, dtype=torch.int32, device=dev) for s in ((F, cap), (F, cap + 1), (F, cap), (F,))]
        d_ids = torch.full((F, cap), -7, dtype=torch.int32, device=dev)
        d_vals = torch.zeros((F, cap), dtype=torch.float64, device=dev)
        d_n = torch.full((F,), -7, dtype=torch.int32, device=dev)
        qrow, cov_ptr, cov_row = np.array([0, 3], np.int32), np.array([0, 2, 4], np.int32), np.array([1, 3, 0, 1], np.int32)
        d_q, d_p, d_r = _t(qrow), _t(cov_ptr), _t(cov_row)
        d_sc = torch.zeros(4, dtype=torch.float64, device=dev)
        d_min = torch.full((2,), float("nan"), dtype=torch.float32, device=dev)
        host_desc = random_descriptors(700, 99)
        for spun in (False, True):     # the calls rewrite their outputs with the same values
            torch.cuda.synchronize()
            if spun:
                _spin(A)
            v.descend_device(d_desc.data_ptr(), F * cap, levelsup, d_leaf.data_ptr(), d_node.data_ptr(), A.cuda_stream)
            Bs.wait_stream(A)                            # the vocabulary orders no calls: B reads what A wrote
            B.feature_vector_device(v, F, d_leaf.data_ptr(), d_node.data_ptr(), d_cnt.data_ptr(), cap, *[x.data_ptr() for x in d_fv],
                                    Bs.cuda_stream)
            host = v.transform(host_desc, levelsup)
            B.bow_vector_device(v, F, d_leaf.data_ptr(), d_cnt.data_ptr(), cap, d_ids.data_ptr(), d_vals.data_ptr(), d_n.data_ptr(),
                                A.cuda_stream)
            B.min_score_device(v, 2, F, cap, d_ids.data_ptr(), d_vals.data_ptr(), d_n.data_ptr(), d_q.data_ptr(), d_p.data_ptr(),
                               d_r.data_ptr(), d_sc.data_ptr(), d_min.data_ptr(), A.cuda_stream)
        torch.cuda.synchronize()
        want_host = O.bow_transform(voc, host_desc, levelsup)
        assert all(np.array_equal(a, b) for a, b in zip(host[0], want_host[0]))
        assert all(np.array_equal(a, b) for a, b in zip(host[1], want_host[1]))
        ids, vals, n = d_ids.cpu().numpy(), d_vals.cpu().numpy(), d_n.cpu().numpy()
        fv = [x.cpu().numpy() for x in d_fv]
        rows = []
        for f in range(F):
            c = int(counts[f])
            (wi, wv), (fi, fp, ft) = O.bow_transform(voc, desc[f, :c], levelsup)
            k = int(n[f])
            assert np.array_equal(ids[f, :k], wi) and np.array_equal(vals[f, :k].view(np.uint64), np.asarray(wv, np.float64).view(np.uint64)), f
            nn = int(fv[3][f])
            assert np.array_equal(fv[0][f, :nn], fi) and np.array_equal(fv[1][f, :nn + 1], fp), f
            assert np.array_equal(fv[2][f, :fv[1][f, nn]], ft), f
            rows.append((wi, wv))
        sc, mn = d_sc.cpu().numpy(), d_min.cpu().numpy()
        for b, q in enumerate(qrow):
            lo = np.float32(1)
            for k in range(cov_ptr[b], cov_ptr[b + 1]):
                s = v.score(*rows[q], *rows[cov_row[k]])
                assert sc[k].view(np.uint64) == np.float64(s).view(np.uint64), (b, k)
                lo = min(lo, np.float32(s))
            assert mn[b].view(np.uint32) == lo.view(np.uint32), b
    finally:
        v.close()
