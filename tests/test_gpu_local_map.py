"""GPU tests of orbfe_covis_local_map_device (Tracking::UpdateReference for one frame): after every step of every scene of
tests/local_map_scenes.py, and for frames of 300, 1000 and 2000 matched points on the 2000 x 2000 map, the device's frame
cells, local keyframes, reference keyframe and local points equal the oracle that tests/test_oracle_local_map.py pins to the
reference's own Tracking.cc, with cells past each row's count holding point indices that must not be read; the rows a
device KeyFrameCulling leaves, with its erases, observations and UpdateConnections, feed a local-map call equal to the
oracle run the same way; malformed input writes nothing and sync reports it once; and the call is ordered after the
handle's work on another stream."""
import numpy as np
import pytest

import orb_slam_b200 as fe
from orb_slam_b200 import bow as B
from oracle import kf_culling as KC
from oracle import local_map as LM
from oracle import observations as OO

import covis_scenes as S
import kf_culling_scenes as KS
import local_map_scenes as LS
from test_gpu_kf_culling import Run as CullRun, _dev, _full, _torch, FILL, SPIN
from test_oracle_local_map import lm_inputs

pytestmark = pytest.mark.gpu


def _past_counts(a, cap):
    """a copy of the inputs whose cells past each row's count name points (they must not be read)"""
    a = {k: np.array(v, copy=True) for k, v in a.items()}
    npts = len(a["point_bad"])
    if npts:
        rows = a["kf_mp"].reshape(-1, cap)
        past = np.arange(cap)[None, :] >= a["counts"][:, None]
        rows[past] = (np.arange(rows.size).reshape(rows.shape) % npts)[past]
    return a


class Run(CullRun):
    """a scene on the device graph, the oracle graph and the model, with local-map calls on both"""

    def __init__(self, scene):
        super().__init__(scene)
        self.model = LS.LmModel(scene)

    def lists(self):
        return {s: self.orc.ordered(s)[0] for s in range(self.K)}

    def oracle(self, cells, a=None):
        a = _past_counts(lm_inputs(self.model, self.slot_of, self.K), self.cap) if a is None else a
        nb, nnb = LM.neighbours(self.lists(), self.K)
        return LM.local_map(cells, a["point_bad"], a["kf_mp"], a["counts"], self.cap, a["live"], a["keys"], nb, nnb), a

    def bufs(self, cells, a):
        npts = len(a["point_bad"])
        return dict(frame=_dev(cells if len(cells) else [0]), point_bad=_dev(a["point_bad"] if npts else [0], np.uint8), kf_mp=_dev(a["kf_mp"]),
                    counts=_dev(a["counts"]), lk=_full(self.K), nlk=_full(1), ref=_full(1), lp=_full(npts), nlp=_full(1))

    def device(self, cells, a, stream=0, sync=True, bufs=None, scr=None, nframes=None):
        """one call; returns every buffer as host arrays, FILL where unwritten.  With the buffers and the scratch given,
        nothing is allocated and nothing synchronised before the call"""
        torch, dev = _torch()
        npts = len(a["point_bad"])
        d = bufs or self.bufs(cells, a)
        if scr is None:
            nb = B.CovisibilityGraph.local_map_scratch_bytes(npts, self.K)
            scr = torch.randint(-2 ** 31, 2 ** 31 - 1, (nb // 4 + 1,), dtype=torch.int32, device=dev)   # contents ignored
            torch.cuda.synchronize()
        self.g.local_map_device(len(cells), d["frame"].data_ptr(), d["point_bad"].data_ptr(), npts, d["kf_mp"].data_ptr(),
                                d["counts"].data_ptr(), self.K if nframes is None else nframes, self.cap, d["lk"].data_ptr(),
                                d["nlk"].data_ptr(), d["ref"].data_ptr(), d["lp"].data_ptr(), d["nlp"].data_ptr(), scr.data_ptr(), stream)
        if sync:
            self.g.sync()
        torch.cuda.synchronize()
        return {k: v.cpu().numpy() for k, v in d.items()}, d

    def check(self, cells, where=None, a=None):
        o, a = self.oracle(cells, a)
        assert o["status"] == 0, where
        got, _ = self.device(cells, a)
        compare(got, o, len(cells), where)
        return o, got


def compare(got, o, nf, where, tails=True):
    """the device's buffers equal the oracle's result; with tails, nothing is written past the counts"""
    nlk, nlp = len(o["local_kf"]), len(o["local_points"])
    assert got["frame"][:nf].tolist() == o["frame_mp"].tolist(), (where, "frame cells")
    assert int(got["nlk"][0]) == nlk and got["lk"][:nlk].tolist() == o["local_kf"].tolist(), (where, "local keyframes")
    assert not tails or (got["lk"][nlk:] == FILL).all(), where
    assert int(got["ref"][0]) == o["ref_kf"], (where, "reference keyframe")
    assert int(got["nlp"][0]) == nlp and got["lp"][:nlp].tolist() == o["local_points"].tolist(), (where, "local points")
    assert not tails or (got["lp"][nlp:] == FILL).all(), where


def _play(scene, check_all=True):
    r = Run(scene)
    try:
        for t, step in enumerate(scene.steps):
            where = (scene.name, t, step[0])
            if step[0] == "frame":
                r.check(step[1], where)
                continue
            if step[0] != "to_be_erased":   # mbToBeErased is no state of the device's
                r.step(step)
            if check_all:
                r.check(LS.probe_frame(r.model), where + ("probe",))
        return r
    except BaseException:
        r.close()
        raise


@pytest.mark.parametrize("scene", LS.small_scenes(), ids=lambda s: s.name)
def test_device_equals_oracle_after_every_step(gpu_required, scene):
    _play(scene).close()


def test_large_map(gpu_required):
    """2000 keyframes x 2000 features: frames of 300, 1000 and 2000 matched points around keyframe 1000"""
    r = _play(S.scene_large(), check_all=False)
    try:
        for cells in LS.large_frames(r.model, r.slot_of):
            o, _ = r.check(cells, ("large", len(cells)))
            assert len(o["local_kf"]) > 10
    finally:
        r.close()


def test_malformed_input_writes_nothing(gpu_required):
    """a frame cell or a live row's value >= npoints, or a live slot's count outside 0 .. cap: sync raises once, and no
    output or frame cell changed; a live slot >= nframes is refused on the host"""
    r = _play(LS.scene_listed_and_limits(), check_all=False)
    try:
        cells = np.array(r.scene.steps[-1][1], np.int32)
        base = _past_counts(lm_inputs(r.model, r.slot_of, r.K), r.cap)
        npts = len(base["point_bad"])
        live = np.flatnonzero(base["live"])
        row0 = int(live[0]) * r.cap

        def run_case(mut_cells, mut):
            a = {k: np.array(v, copy=True) for k, v in base.items()}
            c = np.array(cells, copy=True)
            mut_cells(c)
            mut(a)
            got, _ = r.device(c, a, sync=False)
            with pytest.raises(fe.OrbfeError) as e:
                r.g.sync()
            assert e.value.code == fe.ORBFE_ERR_ARG and b"local map" in fe.lib().orbfe_last_error()
            r.g.sync()   # reported once
            assert got["frame"][:len(c)].tolist() == c.tolist()
            for k in ("lk", "nlk", "ref", "lp", "nlp"):
                assert (got[k] == FILL).all(), k

        run_case(lambda c: c.__setitem__(0, npts), lambda a: None)
        run_case(lambda c: None, lambda a: a["kf_mp"].__setitem__(row0, npts))
        run_case(lambda c: None, lambda a: a["counts"].__setitem__(int(live[-1]), r.cap + 1))
        run_case(lambda c: None, lambda a: a["counts"].__setitem__(int(live[0]), -1))
        with pytest.raises(fe.OrbfeError) as e:
            r.device(cells, base, nframes=int(live.max()))
        assert e.value.code == fe.ORBFE_ERR_ARG and b"live slot" in fe.lib().orbfe_last_error()
        r.check(cells)   # the handle works afterwards
    finally:
        r.close()


def test_chain_rows_cull_erase_observations_update_local_map(gpu_required):
    """KeyFrameCulling on the device, orbfe_covis_erase of the ERASED slots in order, observations_device on the rows the
    cull left, update_connections_device of the current keyframe's neighbours from those lists, then a local-map call on the
    rows and point flags the cull left: equal to the oracle run the same way (the culling oracle's rows and flags, its
    erases, the GetObservations oracle, the covisibility oracle, the local-map oracle)"""
    scene = KS.scene_ref_and_cascade()
    r = Run(scene)
    try:
        for step in scene.steps:
            if step[0] == "cull":
                break
            r.step(step)
        cur = step[1]
        o, a = CullRun.oracle(r, cur)
        got, d = CullRun.device(r, cur, a=a)
        erased = [int(v) for v, c in zip(o["verdict_slot"], o["verdict"]) if c == KC.ERASED]
        assert erased and got["vd"][:len(o["verdict"])].tolist() == o["verdict"].tolist()
        for s in erased:
            r.erase(s)
        live = a["live"].copy()
        live[erased] = 0
        npts = len(a["point_bad"])
        allp = np.arange(npts, dtype=np.int32)
        rc, optr, oobs, onobs, _ = OO.observations(allp, npts, o["kf_mp"], a["counts"], r.cap, live, a["keys"])
        assert rc == 0
        d_ptr, d_obs, d_nobs = _full(npts + 1), _full(max(onobs, 1)), _full(1)
        scr = _full(B.CovisibilityGraph.observations_scratch_bytes(npts, r.K, r.cap, onobs) // 4 + 1, 0)
        r.g.observations_device(npts, _dev(allp).data_ptr(), npts, d["kf_mp"].data_ptr(), d["counts"].data_ptr(), r.K, r.cap, onobs,
                                d_ptr.data_ptr(), d_obs.data_ptr(), d_nobs.data_ptr(), scr.data_ptr())
        r.g.sync()
        nb = [int(s) for s in r.orc.ordered(int(r.slot_of[cur]))[0] if r.orc.live(int(s))]
        r.orc.replay(nb, o["kf_mp"], a["counts"], r.cap, optr, oobs)
        r.g.update_connections_device(nb, d["kf_mp"].data_ptr(), d["counts"].data_ptr(), r.K, r.cap, d_ptr.data_ptr(), d_obs.data_ptr(),
                                      npts, onobs)
        r.g.sync()
        cells = np.array([p for p in range(npts)] + [0, 1], np.int32)   # every point, bad ones included, two of them twice
        la = dict(kf_mp=o["kf_mp"], counts=a["counts"], live=live, keys=a["keys"], point_bad=o["point_bad"])
        lo, _ = r.oracle(cells, la)
        assert lo["status"] == 0 and len(lo["local_kf"]) > 1
        bufs = dict(frame=_dev(cells), point_bad=d["point_bad"], kf_mp=d["kf_mp"], counts=d["counts"], lk=_full(r.K), nlk=_full(1),
                    ref=_full(1), lp=_full(npts), nlp=_full(1))
        lgot, _ = r.device(cells, la, bufs=bufs)
        compare(lgot, lo, len(cells), "chain")
    finally:
        r.close()


def test_ordered_after_graph_work_on_another_stream(gpu_required):
    """observations_device enqueued on stream A behind a spin writes its list pointers into the local-keyframe buffer the
    local-map call then gets on stream B, enqueued right after it with nothing synchronised in between (observations_device
    copies nothing from the host, so the host does not wait for the spin): the local-map call runs after it, so the buffer
    holds the local keyframes, not the pointers"""
    torch, dev = _torch()
    r = _play(LS.scene_bound(79), check_all=False)
    try:
        cells = np.array(r.scene.steps[-1][1], np.int32)
        o, a = r.oracle(cells)
        assert len(o["local_kf"]) == 81
        npts = len(a["point_bad"])
        bufs = r.bufs(cells, a)
        scr = _full(B.CovisibilityGraph.local_map_scratch_bytes(npts, r.K) // 4 + 1, 0)
        nobs = int(np.count_nonzero(a["kf_mp"] >= 0))
        m = min(npts, r.K - 1)                        # its d_ptr (m + 1 entries) fits the local-keyframe buffer
        d_pts, o_obs, o_nobs = _dev(np.arange(m)), _full(nobs), _full(1)
        o_scr = _full(B.CovisibilityGraph.observations_scratch_bytes(npts, r.K, r.cap, nobs) // 4 + 1, 0)
        d_kf_mp = _dev(lm_inputs(r.model, r.slot_of, r.K)["kf_mp"])
        A, Bs = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)
        torch.cuda.synchronize()   # everything allocated and uploaded; from here on only enqueues until the sync
        with torch.cuda.stream(A):
            torch.cuda._sleep(SPIN)
        r.g.observations_device(m, d_pts.data_ptr(), npts, d_kf_mp.data_ptr(), bufs["counts"].data_ptr(), r.K, r.cap, nobs,
                                bufs["lk"].data_ptr(), o_obs.data_ptr(), o_nobs.data_ptr(), o_scr.data_ptr(), stream=A.cuda_stream)
        got, _ = r.device(cells, a, stream=Bs.cuda_stream, bufs=bufs, scr=scr)
        compare(got, o, len(cells), "stream order", tails=False)
    finally:
        r.close()
