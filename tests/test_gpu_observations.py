"""GPU tests of orbfe_covis_observations_device (MapPoint::GetObservations() built from the keyframes' rows): after every
step of every scene of tests/observation_scenes.py and tests/covis_scenes.py, and on the 2000 x 2000 map, the device lists,
pointers, total and ref_obs equal the oracle that tests/test_oracle_observations.py pins to the reference, for all points
and for named subsets in any order (a subset's groups equal the same groups of the all-points call); overflow, a point
named twice or out of range, a bad count, a row value or reference slot out of range leave only d_ptr (and on overflow
*d_nobs) written and are reported by sync; the call is ordered after graph work on another stream; and rows ->
observations_device -> distinctive_descriptors_device + normal_and_depth_device + update_connections_device equals the
same three calls fed the host lists."""
import numpy as np
import pytest

import orb_slam_b200 as fe
from orb_slam_b200 import bow as B
from oracle import observations as OO

import covis_scenes as S
import observation_scenes as OS
from test_oracle_observations import oracle_inputs

pytestmark = pytest.mark.gpu
SPIN = 100_000_000          # torch.cuda._sleep cycles: one bounded spin of roughly 50 ms on an H100
FILL = -7


def _torch():
    import torch
    return torch, torch.device("cuda", 0)


def _dev(a, dt=np.int32):
    torch, dev = _torch()
    return torch.from_numpy(np.ascontiguousarray(a, dt)).to(dev)


def _full(n, v=FILL):
    torch, dev = _torch()
    return torch.full((max(int(n), 1),), v, dtype=torch.int32, device=dev)


class Run:
    """A scene on the device graph (a keyframe is added when it becomes an observer, erased with KeyFrame::SetBadFlag) and
    on the model the oracle reads."""

    def __init__(self, scene):
        self.scene, self.K, self.cap = scene, scene.nkf, scene.cap
        self.slot_of = scene.slots()
        self.model = OS.ObsModel(scene)
        self.g = B.CovisibilityGraph(self.K, scene.max_connections, 64)
        self._dv = None

    def close(self):
        self.g.close()

    def step(self, step):
        self.model.apply(step)
        op = step[0]
        if op == "kf" or op == "process":
            k = len(self.model.nfeat) - 1 if op == "kf" else step[1]
            self.g.add([int(self.slot_of[k])], [k], [k])
        elif op == "erase_kf":
            self.g.erase(int(self.slot_of[step[1]]))

    def inputs(self):
        kf_mp, counts, gp, obs, live, keys, ref_slot = oracle_inputs(self.model, self.slot_of, self.K)
        if self._dv is None or self._dv[0] != self.model.version:
            self._dv = (self.model.version, _dev(kf_mp), _dev(counts))
        return (kf_mp, counts, gp, obs, live, keys, ref_slot), self._dv[1:]

    def device(self, points, ref_slot=None, obs_cap=None, npoints=None, d_rows=None, nframes=None, stream=0, sync=True, out=None):
        """one call; returns (ptr, obs buffer, nobs, ref_obs buffer) as host arrays (the whole buffers, FILL where unwritten)"""
        torch, dev = _torch()
        (kf_mp, *_), (d_mp, d_cnt) = self.inputs()
        if d_rows is not None:
            d_mp, d_cnt = d_rows
        npoints = len(self.model.obs) if npoints is None else npoints
        obs_cap = int(np.count_nonzero(kf_mp >= 0)) if obs_cap is None else obs_cap
        n = len(points)
        d_pts = _dev(points if n else [0])
        d_ptr, d_obs, d_nobs = (_full(n + 1), _full(obs_cap), _full(1)) if out is None else out
        d_rs = _dev(ref_slot if len(ref_slot) else [0]) if ref_slot is not None else None
        d_ro = _full(n) if ref_slot is not None else None
        nb = B.CovisibilityGraph.observations_scratch_bytes(npoints, self.K, self.cap, obs_cap)
        d_scr = torch.randint(-2 ** 31, 2 ** 31 - 1, (nb // 4 + 1,), dtype=torch.int32, device=dev)   # contents ignored
        torch.cuda.synchronize()
        self.g.observations_device(n, d_pts.data_ptr(), npoints, d_mp.data_ptr(), d_cnt.data_ptr(), self.K if nframes is None else nframes,
                                   self.cap, obs_cap, d_ptr.data_ptr(), d_obs.data_ptr(), d_nobs.data_ptr(), d_scr.data_ptr(),
                                   0 if d_rs is None else d_rs.data_ptr(), 0 if d_ro is None else d_ro.data_ptr(), stream)
        if sync:
            self.g.sync()
        torch.cuda.synchronize()
        return (d_ptr.cpu().numpy(), d_obs.cpu().numpy(), int(d_nobs.cpu().numpy()[0]),
                None if d_ro is None else d_ro.cpu().numpy()[:n])

    def check(self, where, rng):
        (kf_mp, counts, gp, obs, live, keys, ref_slot), _ = self.inputs()
        npts = len(self.model.obs)
        allp = np.arange(npts, dtype=np.int32)
        rc, optr, oobs, onobs, oref = OO.observations(allp, npts, kf_mp, counts, self.cap, live, keys, ref_slot)
        assert rc == 0
        ptr, dobs, nobs, ref = self.device(allp, ref_slot)
        assert ptr.tolist() == optr.tolist() and nobs == onobs, where
        assert dobs[:nobs].tolist() == oobs.tolist() and (dobs[nobs:] == FILL).all(), where
        assert ref.tolist() == oref.tolist(), where
        if npts == 0:
            return
        sub = rng.permutation(npts)[:max(1, npts // 2)].astype(np.int32)   # a named subset in a random order
        rc, sptr, sobs, _, sref = OO.observations(sub, npts, kf_mp, counts, self.cap, live, keys, ref_slot[sub])
        p2, d2, n2, r2 = self.device(sub, ref_slot[sub])
        assert p2.tolist() == sptr.tolist() and d2[:n2].tolist() == sobs.tolist() and r2.tolist() == sref.tolist(), where
        for j, m in enumerate(sub.tolist()):
            assert d2[p2[j]:p2[j + 1]].tolist() == dobs[ptr[m]:ptr[m + 1]].tolist(), (where, m)


SCENES = OS.small_scenes() + S.small_scenes()


@pytest.mark.parametrize("scene", SCENES, ids=lambda s: s.name)
def test_device_equals_oracle_after_every_step(gpu_required, scene):
    r = Run(scene)
    rng = np.random.default_rng(7)
    try:
        for t, step in enumerate(scene.steps):
            r.step(step)
            r.check((scene.name, t, step[0]), rng)
    finally:
        r.close()


@pytest.fixture(scope="module")
def large():
    return S.scene_large()


def _run_large(large):
    r = Run(large)
    for step in large.steps:
        r.step(step)
    return r


def test_large_map(gpu_required, large):
    """2000 keyframes x 2000 features: all points, the points of one keyframe's row, and a random half"""
    r = _run_large(large)
    try:
        r.check("large", np.random.default_rng(8))
        (kf_mp, counts, _, _, live, keys, ref_slot), _ = r.inputs()
        s = int(r.slot_of[1000])
        pts = np.unique(kf_mp[s * r.cap:(s + 1) * r.cap])
        pts = pts[pts >= 0].astype(np.int32)
        rc, optr, oobs, _, oref = OO.observations(pts, len(r.model.obs), kf_mp, counts, r.cap, live, keys, ref_slot[pts])
        ptr, dobs, nobs, ref = r.device(pts, ref_slot[pts])
        assert ptr.tolist() == optr.tolist() and dobs[:nobs].tolist() == oobs.tolist() and ref.tolist() == oref.tolist()
    finally:
        r.close()


def test_long_lists(gpu_required):
    """points seen by 33, 64, 1500 and 2047 keyframes (the block-ranked path, keys tiled past 1024), slots a permutation"""
    s = OS.ObsScene("long", 8, seed=31, max_connections=2048)
    ks = [s.kf() for _ in range(2048)]
    obs = []
    for j, width in enumerate((33, 64, 1500, 2047, 3, 32)):
        obs += [(j, k, j) for k in ks[:width]]
    s.pts([0] * 6, obs)
    for k in range(0, 2048, 7):
        s.row(k, 7, 3)   # point 3 again at feature 7 of every seventh keyframe: the larger index
    r = Run(s)
    try:
        for step in s.steps:
            r.step(step)
        r.check("long", np.random.default_rng(9))
    finally:
        r.close()


def _error_scene():
    r = Run(OS.scene_fuse())
    for step in r.scene.steps:
        r.step(step)
    return r


def test_overflow_writes_ptr_and_the_size_needed(gpu_required):
    r = _error_scene()
    try:
        (kf_mp, counts, gp, obs, live, keys, ref_slot), _ = r.inputs()
        allp = np.arange(len(r.model.obs), dtype=np.int32)
        _, optr, _, onobs, _ = OO.observations(allp, len(allp), kf_mp, counts, r.cap, live, keys, ref_slot)
        with pytest.raises(fe.OrbfeError) as e:
            r.device(allp, ref_slot, obs_cap=onobs - 1)
        assert e.value.code == fe.ORBFE_ERR_CAPACITY
        ptr, dobs, nobs, ref = r.device(allp, ref_slot, obs_cap=onobs - 1, sync=False)
        assert ptr.tolist() == optr.tolist() and nobs == onobs
        assert (dobs == FILL).all() and (ref == FILL).all()
        with pytest.raises(fe.OrbfeError):
            r.g.sync()
        r.g.sync()   # reported once
        ptr, dobs, nobs, ref = r.device(allp, ref_slot, obs_cap=onobs)   # exactly enough
        assert nobs == onobs and ptr.tolist() == optr.tolist()
    finally:
        r.close()


def test_bad_input_writes_only_ptr(gpu_required):
    r = _error_scene()
    torch, dev = _torch()
    try:
        (kf_mp, counts, gp, obs, live, keys, ref_slot), (d_mp, d_cnt) = r.inputs()
        npts = len(r.model.obs)
        allp = np.arange(npts, dtype=np.int32)
        s_live = int(np.nonzero(live)[0][0])
        c2 = counts.copy()
        c2[s_live] = r.cap + 1
        cases = [
            ("point named twice", dict(points=np.array([0, 1, 0], np.int32))),
            ("point out of range", dict(points=np.array([0, npts], np.int32), npoints=npts)),
            ("negative point", dict(points=np.array([-1], np.int32))),
            ("count > cap", dict(points=allp, d_rows=(d_mp, _dev(c2)))),
            ("row value >= npoints", dict(points=allp[:2], npoints=int(kf_mp.max()))),
            ("reference slot out of range", dict(points=allp[:2], ref_slot=np.array([0, r.K], np.int32))),
        ]
        for name, kw in cases:
            pts = kw.pop("points")
            ref = kw.pop("ref_slot", ref_slot[np.clip(pts, 0, npts - 1)])
            with pytest.raises(fe.OrbfeError) as e:
                r.device(pts, ref, **kw)
            assert e.value.code == fe.ORBFE_ERR_ARG, name
            ptr, dobs, nobs, ro = r.device(pts, ref, sync=False, **kw)
            with pytest.raises(fe.OrbfeError):
                r.g.sync()
            assert (dobs == FILL).all() and nobs == FILL and (ro == FILL).all(), name
            assert ptr[0] == 0, name
        r.check("after the errors", np.random.default_rng(3))
        # host-side: a live slot >= nframes, before the handle is used
        with pytest.raises(fe.OrbfeError) as e:
            r.device(allp, ref_slot, nframes=int(np.nonzero(live)[0].max()))
        assert e.value.code == fe.ORBFE_ERR_ARG and "nframes" in str(e.value)
        r.g.sync()
    finally:
        r.close()


def test_ordered_after_graph_work_on_another_stream(gpu_required):
    """lists_device enqueued on stream A behind a spin writes into the buffers the observations call then gets on stream B:
    the observations call runs after it, so the buffers hold its result"""
    torch, dev = _torch()
    r = _error_scene()
    try:
        (kf_mp, counts, gp, obs, live, keys, ref_slot), (d_mp, d_cnt) = r.inputs()
        n = len(r.model.obs)
        allp = np.arange(n, dtype=np.int32)
        _, optr, oobs, onobs, oref = OO.observations(allp, n, kf_mp, counts, r.cap, live, keys, ref_slot)
        big = max(n + 1, n * r.g.max_connections, onobs)
        d_ptr, d_obs, d_nobs, d_ro = _full(big), _full(big), _full(1), _full(n)
        d_pts, d_rs = _dev(allp), _dev(ref_slot)
        d_scr = _full(B.CovisibilityGraph.observations_scratch_bytes(n, r.K, r.cap, onobs) // 4 + 1, 0)
        A, Bs = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)
        slots = list(range(min(n, r.K)))   # its d_ptr overlaps the one the observations call writes
        torch.cuda.synchronize()
        with torch.cuda.stream(A):
            torch.cuda._sleep(SPIN)
        r.g.lists_device(1, slots, 0, d_ptr.data_ptr(), d_obs.data_ptr(), stream=A.cuda_stream)
        r.g.observations_device(n, d_pts.data_ptr(), n, d_mp.data_ptr(), d_cnt.data_ptr(), r.K, r.cap, onobs, d_ptr.data_ptr(),
                                d_obs.data_ptr(), d_nobs.data_ptr(), d_scr.data_ptr(), d_rs.data_ptr(), d_ro.data_ptr(), Bs.cuda_stream)
        r.g.sync()
        torch.cuda.synchronize()
        ptr, dobs = d_ptr.cpu().numpy(), d_obs.cpu().numpy()
        assert ptr[:n + 1].tolist() == optr.tolist() and int(d_nobs.item()) == onobs and dobs[:onobs].tolist() == oobs.tolist()
        assert d_ro.cpu().numpy().tolist() == oref.tolist()
    finally:
        r.close()


def _chain(run, d_ptr, d_obs, nobs, d_ref_obs, rng_seed):
    """distinctive_descriptors_device + normal_and_depth_device + update_connections_device of every live slot on the lists"""
    torch, dev = _torch()
    K, cap, npts = run.K, run.cap, len(run.model.obs)
    rng = np.random.default_rng(rng_seed)
    (kf_mp, counts, *_), (d_mp, d_cnt) = run.inputs()
    desc = _dev(rng.integers(0, 256, (K * cap, 32)), np.uint8)
    kps = np.zeros(K * cap, fe.KP_DTYPE)
    kps["octave"] = rng.integers(0, 8, K * cap)
    d_kps = _dev(kps.view(np.uint8), np.uint8)
    d_c = _dev(rng.standard_normal((K, 3)), np.float32)
    d_w = _dev(rng.standard_normal((max(npts, 1), 3)) + 5, np.float32)
    m = fe.ORBmatcher(0.6, True)
    d_best = _full(npts, -9)
    d_mpd = torch.zeros((max(npts, 1), 32), dtype=torch.uint8, device=dev)
    f32 = lambda *s: torch.full(s, 0.5, dtype=torch.float32, device=dev)
    d_n, d_a, d_b = f32(max(npts, 1), 3), f32(max(npts, 1)), f32(max(npts, 1))
    sfs = (1.2 ** np.arange(8)).astype(np.float32)
    torch.cuda.synchronize()
    B.distinctive_descriptors_device(m, npts, desc.data_ptr(), d_cnt.data_ptr(), K, cap, d_ptr.data_ptr(), d_obs.data_ptr(), nobs,
                                     d_best.data_ptr(), d_mpd.data_ptr())
    B.normal_and_depth_device(m, npts, d_kps.data_ptr(), d_cnt.data_ptr(), K, cap, d_c.data_ptr(), d_ptr.data_ptr(), d_obs.data_ptr(), nobs,
                              d_w.data_ptr(), d_ref_obs.data_ptr(), 1.2, sfs, d_n.data_ptr(), d_a.data_ptr(), d_b.data_ptr())
    m.sync()
    g = B.CovisibilityGraph(K, 2048, 64)
    live = [k for k in range(len(run.model.nfeat)) if run.model.live()[k]]
    slots = [int(run.slot_of[k]) for k in live]
    try:
        if slots:
            g.add(slots, live, live)
            for i in range(0, len(slots), 64):
                g.update_connections_device(slots[i:i + 64], d_mp.data_ptr(), d_cnt.data_ptr(), K, cap, d_ptr.data_ptr(), d_obs.data_ptr(),
                                            npts, nobs)
            g.sync()
        from test_gpu_covis import state
        graph = state(g, K)
    finally:
        g.close()
        m.close()
    return (d_best.cpu().numpy(), d_mpd.cpu().numpy(), d_n.cpu().numpy().view(np.int32), d_a.cpu().numpy().view(np.int32),
            d_b.cpu().numpy().view(np.int32), graph)


def _chain_equal(run):
    torch, dev = _torch()
    (kf_mp, counts, gp, obs, live, keys, ref_slot), _ = run.inputs()
    npts = len(run.model.obs)
    cap = run.cap
    host_ref = np.array([ref_slot[m] * cap + run.model.obs[m].get(run.model.ref[m], 0) if run.model.ref[m] >= 0 else ref_slot[m] * cap
                         for m in range(npts)], np.int32)
    host = _chain(run, _dev(gp), _dev(obs if len(obs) else [0]), len(obs), _dev(host_ref if npts else [0]), 5)
    allp = np.arange(npts, dtype=np.int32)
    obs_cap = int(np.count_nonzero(kf_mp >= 0))
    out = (_full(npts + 1), _full(obs_cap), _full(1))
    d_rs, d_ro = _dev(ref_slot if npts else [0]), _full(npts)
    nb = B.CovisibilityGraph.observations_scratch_bytes(npts, run.K, cap, obs_cap)
    d_scr = _full(nb // 4 + 1, 0)
    (_, (d_mp, d_cnt)) = run.inputs()
    torch.cuda.synchronize()
    run.g.observations_device(npts, _dev(allp if npts else [0]).data_ptr(), npts, d_mp.data_ptr(), d_cnt.data_ptr(), run.K, cap, obs_cap,
                              out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(), d_scr.data_ptr(), d_rs.data_ptr(), d_ro.data_ptr())
    run.g.sync()
    nobs = int(out[2].cpu().numpy()[0])
    assert nobs == len(obs)
    dev_ = _chain(run, out[0], out[1], nobs, d_ro, 5)
    for a, b in zip(host[:5], dev_[:5]):
        assert np.array_equal(a, b)
    assert host[5] == dev_[5]


@pytest.mark.parametrize("scene", OS.small_scenes()[:-1], ids=lambda s: s.name)
def test_chain_equals_host_lists(gpu_required, scene):
    r = Run(scene)
    try:
        for step in scene.steps:
            r.step(step)
        _chain_equal(r)
    finally:
        r.close()


def test_chain_equals_host_lists_large_map(gpu_required, large):
    r = _run_large(large)
    try:
        _chain_equal(r)
    finally:
        r.close()


def test_cells_past_the_count_are_not_read(gpu_required):
    """rows whose cells past d_counts[s] still name points: only i < d_counts[s] is read"""
    r = _error_scene()
    try:
        (kf_mp, counts, gp, obs, live, keys, ref_slot), (d_mp, _) = r.inputs()
        c2 = counts.copy()
        c2[live.astype(bool)] = np.maximum(c2[live.astype(bool)] - 59, 0)   # keeps features 0..4 of a 64-feature row
        n = len(r.model.obs)
        allp = np.arange(n, dtype=np.int32)
        assert any((kf_mp.reshape(r.K, r.cap)[s, c2[s]:] >= 0).any() for s in range(r.K) if live[s])
        _, optr, oobs, onobs, oref = OO.observations(allp, n, kf_mp, c2, r.cap, live, keys, ref_slot)
        ptr, dobs, nobs, ref = r.device(allp, ref_slot, d_rows=(d_mp, _dev(c2)))
        assert ptr.tolist() == optr.tolist() and dobs[:nobs].tolist() == oobs.tolist() and ref.tolist() == oref.tolist()
    finally:
        r.close()
