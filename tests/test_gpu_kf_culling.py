"""GPU tests of orbfe_covis_keyframe_culling_device (LocalMapping::KeyFrameCulling with SetBadFlag's map-point half): after
every step of every scene of tests/kf_culling_scenes.py, and on the 2000 x 2000 map, the device's verdicts, nMPs,
nRedundant, rows, point flags, reference slots and made-bad points equal the oracle that tests/test_oracle_kf_culling.py pins
to the reference's own LocalMapping.cc; the rows it leaves, with the ERASED keyframes erased from the graph in order, feed
observations_device, update_connections_device and lists_device to the oracle's results; malformed input and an obs_cap
overflow write nothing (but *d_nobs on overflow) and sync reports the code; and the call is ordered after the handle's work
on another stream."""
import numpy as np
import pytest

import orb_slam_b200 as fe
from orb_slam_b200 import bow as B
from oracle import kf_culling as KC
from oracle import observations as OO
from oracle.covis import CovisOracle

import covis_key_scenes as KM
import covis_scenes as S
import kf_culling_scenes as KS
from test_oracle_kf_culling import cull_inputs

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


def _kps(octave):
    kp = np.zeros(len(octave), fe.KP_DTYPE)
    kp["octave"] = octave
    return _dev(kp.view(np.uint8), np.uint8)


class Run:
    """A scene on the device graph and the oracle graph (keyframes added when they become observers), on the model, and
    the culls on both.  keys[k] is keyframe k's order key (the creation index when None)."""

    def __init__(self, scene, keys=None, max_batch=64):
        self.scene, self.K, self.cap, self.keys = scene, scene.nkf, scene.cap, keys
        self.slot_of = scene.slots()
        self.model = KS.CullModel(scene, keys)
        self.g = B.CovisibilityGraph(self.K, scene.max_connections, max_batch)
        self.orc = CovisOracle(self.K)

    def close(self):
        self.g.close()
        self.orc.close()

    def add(self, k):
        s = int(self.slot_of[k])
        self.g.add([s], [k], [KM.key_of(self.keys, k)])
        self.orc.add(s, k, KM.key_of(self.keys, k))

    def erase(self, s):
        self.g.erase(s)
        self.orc.erase(s)

    def step(self, step, erased=()):
        self.model.apply(step, erased=erased)
        op = step[0]
        if op == "kf":
            self.add(len(self.model.nfeat) - 1)
        elif op == "process":
            self.add(step[1])
        elif op == "erase_kf":
            self.erase(int(self.slot_of[step[1]]))
        elif op == "update":
            slots = [int(self.slot_of[k]) for k in step[1]]
            kf_mp, counts, gp, obs = self.model.inputs(self.slot_of, self.K)
            self.orc.replay(slots, kf_mp, counts, self.cap, gp, obs)
            d = [_dev(kf_mp), _dev(counts), _dev(gp), _dev(obs if len(obs) else [0])]
            for i in range(0, len(slots), self.g.max_batch):
                self.g.update_connections_device(slots[i:i + self.g.max_batch], d[0].data_ptr(), d[1].data_ptr(), self.K, self.cap, d[2].data_ptr(),
                                                 d[3].data_ptr(), len(gp) - 1, len(obs))
            self.g.sync()

    def oracle(self, cur, not_erase=(), a=None, obs_cap=None):
        a = cull_inputs(self.model, self.slot_of, self.K, not_erase, self.keys) if a is None else a
        cand = np.array(self.orc.ordered(int(self.slot_of[cur]))[0], np.int32)
        return KC.cull(cand, a["live"], a["id0"], a["keys"], a["not_erase"], a["kf_mp"], a["counts"], a["octave"], self.cap,
                       a["point_bad"], a["ref_slot"], obs_cap=obs_cap), a

    def device(self, cur, not_erase=(), a=None, obs_cap=None, stream=0, sync=True, bufs=None, scr=None):
        """one call on the model's arrays (or `a`); returns every buffer as host arrays, FILL where unwritten.  With the
        buffers and the scratch given, nothing is allocated and the device is not synchronised before the call, so the call
        is enqueued right behind whatever the caller enqueued last"""
        torch, dev = _torch()
        a = cull_inputs(self.model, self.slot_of, self.K, not_erase, self.keys) if a is None else a
        npts = len(a["point_bad"])
        if obs_cap is None:
            obs_cap = int(np.count_nonzero(a["kf_mp"] >= 0))
        C = self.g.max_connections
        d = bufs or dict(kf_mp=_dev(a["kf_mp"]), counts=_dev(a["counts"]), kps=_kps(a["octave"]),
                         point_bad=_dev(a["point_bad"] if npts else [0], np.uint8), ref_slot=_dev(a["ref_slot"] if npts else [0]),
                         nobs=_full(1), vs=_full(C), vd=_full(C), ncand=_full(1), nm=_full(C), nr=_full(C), bp=_full(npts), nbad=_full(1))
        if bufs is None or scr is None:
            nb = B.CovisibilityGraph.cull_scratch_bytes(npts, self.K, self.cap, obs_cap)
            scr = torch.randint(-2 ** 31, 2 ** 31 - 1, (nb // 4 + 1,), dtype=torch.int32, device=dev)   # contents ignored
            torch.cuda.synchronize()
        self.g.keyframe_culling_device(int(self.slot_of[cur]), d["kf_mp"].data_ptr(), d["counts"].data_ptr(), d["kps"].data_ptr(), self.K,
                                       self.cap, d["point_bad"].data_ptr(), d["ref_slot"].data_ptr(), npts,
                                       [int(self.slot_of[k]) for k in not_erase], obs_cap, d["nobs"].data_ptr(), d["vs"].data_ptr(),
                                       d["vd"].data_ptr(), d["ncand"].data_ptr(), d["bp"].data_ptr(), d["nbad"].data_ptr(), scr.data_ptr(),
                                       d["nm"].data_ptr(), d["nr"].data_ptr(), stream)
        if sync:
            self.g.sync()
        torch.cuda.synchronize()
        return {k: v.cpu().numpy() for k, v in d.items()}, d

    def check(self, cur, not_erase=(), where=None):
        """device == oracle on the current map; returns the oracle's result"""
        o, a = self.oracle(cur, not_erase)
        assert o["status"] == 0, where
        got, _ = self.device(cur, not_erase, a)
        n = len(o["verdict"])
        assert int(got["ncand"][0]) == n and int(got["nobs"][0]) == o["nobs"], where
        assert got["vs"][:n].tolist() == o["verdict_slot"].tolist(), where
        assert got["vd"][:n].tolist() == o["verdict"].tolist(), where
        assert got["nm"][:n].tolist() == o["nmps"].tolist() and got["nr"][:n].tolist() == o["nred"].tolist(), where
        assert (got["vs"][n:] == FILL).all() and (got["vd"][n:] == FILL).all(), where
        assert (got["kf_mp"] == o["kf_mp"]).all(), (where, "rows")
        npts = len(a["point_bad"])
        assert (got["point_bad"][:npts] == o["point_bad"]).all() and (got["ref_slot"][:npts] == o["ref_slot"]).all(), where
        nbad = int(got["nbad"][0])
        assert got["bp"][:nbad].tolist() == o["bad_points"].tolist(), where
        return o, got


def _play(scene, check_all=True, keys=None):
    """every step on the device and the oracle; after each step keyframe 1 (the scenes' current keyframe) is culled on both
    without applying it, and a cull step applies the oracle's erases to the model and the graphs"""
    r = Run(scene, keys)
    try:
        for t, step in enumerate(scene.steps):
            where = (scene.name, t, step[0])
            if step[0] == "cull":
                o, _ = r.check(step[1], step[2], where)
                erased = [int(v) for v, c in zip(o["verdict_slot"], o["verdict"]) if c == KC.ERASED]
                kf_of = {int(s): k for k, s in enumerate(r.slot_of)}
                r.step(step, erased=[kf_of[s] for s in erased])
                for s in erased:
                    r.erase(s)
                continue
            r.step(step)
            if check_all and len(r.model.nfeat) > 1 and r.model.live()[1]:
                r.check(1, where=where)
        return r
    except BaseException:
        r.close()
        raise


@pytest.mark.parametrize("scene", KS.small_scenes(), ids=lambda s: s.name)
def test_device_equals_oracle_after_every_step(gpu_required, scene):
    _play(scene).close()


def test_large_map(gpu_required):
    """2000 keyframes x 2000 features: culls for keyframes 1000 and 500, applied in turn"""
    _play(KS.large_culls(S.scene_large()), check_all=False).close()


def test_chain_rows_erase_observations_update_lists(gpu_required):
    """cull on the device, then orbfe_covis_erase of the ERASED slots in order, then observations_device on the rows the
    cull left, update_connections_device of the current keyframe's neighbours from those lists, and lists_device: all equal
    the oracle run the same way (the oracle's rows, its erases, the GetObservations oracle, the covisibility oracle)"""
    torch, dev = _torch()
    scene = KS.scene_ref_and_cascade()
    r = Run(scene)
    try:
        for step in scene.steps:
            if step[0] == "cull":
                break
            r.step(step)
        cur = step[1]
        o, a = r.oracle(cur)
        got, d = r.device(cur, a=a)
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
        assert d_ptr.cpu().numpy().tolist() == optr.tolist() and d_obs.cpu().numpy()[:onobs].tolist() == oobs.tolist()
        nb = [int(s) for s in r.orc.ordered(int(r.slot_of[cur]))[0] if r.orc.live(int(s))]
        r.orc.replay(nb, o["kf_mp"], a["counts"], r.cap, optr, oobs)
        r.g.update_connections_device(nb, d["kf_mp"].data_ptr(), d["counts"].data_ptr(), r.K, r.cap, d_ptr.data_ptr(), d_obs.data_ptr(),
                                      npts, onobs)
        r.g.sync()
        for s in range(r.K):
            want = r.orc.ordered(s)[0]
            d_lp, d_l = _full(2), _full(r.g.max_connections)
            r.g.lists_device(0, [s], 0, d_lp.data_ptr(), d_l.data_ptr())
            r.g.sync()
            n = int(d_lp.cpu().numpy()[1])
            assert [v for v in d_l.cpu().numpy()[:n].tolist()] == [v if r.orc.live(v) else -1 for v in want], s
    finally:
        r.close()


def test_malformed_input_and_overflow_write_nothing(gpu_required):
    """each case: sync raises with its code, and no output or in/out array changed (*d_nobs holds the size needed on
    overflow)"""
    r = _play(KS.scene_order(), check_all=False)
    try:
        cur = 1
        base = cull_inputs(r.model, r.slot_of, r.K)
        need = r.oracle(cur, a=base)[0]["nobs"]
        c_slot = int(r.slot_of[cur])
        cand = r.orc.ordered(c_slot)[0]
        row0 = cand[0] * r.cap

        def run_case(mut, code, obs_cap=None):
            a = {k: np.array(v, copy=True) for k, v in base.items()}
            mut(a)
            got, _ = r.device(cur, a=a, obs_cap=obs_cap, sync=False)
            with pytest.raises(fe.OrbfeError) as e:
                r.g.sync()
            assert e.value.code == code
            npts = len(a["point_bad"])
            assert (got["kf_mp"] == a["kf_mp"]).all() and (got["point_bad"][:npts] == a["point_bad"]).all()
            assert (got["ref_slot"][:npts] == a["ref_slot"]).all()
            for k in ("vs", "vd", "ncand", "nm", "nr", "bp", "nbad"):
                assert (got[k] == FILL).all(), k
            return got

        got = run_case(lambda a: None, fe.ORBFE_ERR_CAPACITY, obs_cap=need - 1)
        assert int(got["nobs"][0]) == need
        for mut in (lambda a: a["counts"].__setitem__(cand[1], r.cap + 1),            # a listed / live slot's count
                    lambda a: a["kf_mp"].__setitem__(row0, len(a["point_bad"])),       # a row value >= npoints
                    lambda a: a["octave"].__setitem__(row0, 32),                       # a listed keyframe's octave
                    lambda a: a["ref_slot"].__setitem__(int(a["kf_mp"][row0]), r.K)):  # a named point's reference slot
            got = run_case(mut, fe.ORBFE_ERR_ARG)
            assert (got["nobs"] == FILL).all() or int(got["nobs"][0]) == need
        r.check(cur)   # the handle works afterwards
    finally:
        r.close()


def test_ordered_after_graph_work_on_another_stream(gpu_required):
    """observations_device enqueued on stream A behind a spin writes its list pointers into the verdict-slot buffer the
    culling call then gets on stream B, enqueued right after it with nothing synchronised in between (observations_device
    copies nothing from the host, so the host does not wait for the spin): the culling call runs after it, so the buffer
    holds the verdict slots, not the pointers"""
    torch, dev = _torch()
    r = _play(KS.scene_stale(), check_all=False)
    try:
        cur = 1
        o, a = r.oracle(cur)
        n = len(o["verdict"])
        C = r.g.max_connections
        npts = len(a["point_bad"])
        bufs = dict(kf_mp=_dev(a["kf_mp"]), counts=_dev(a["counts"]), kps=_kps(a["octave"]), point_bad=_dev(a["point_bad"], np.uint8),
                    ref_slot=_dev(a["ref_slot"]), nobs=_full(1), vs=_full(C), vd=_full(C), ncand=_full(1), nm=_full(C), nr=_full(C),
                    bp=_full(npts), nbad=_full(1))
        scr = _full(B.CovisibilityGraph.cull_scratch_bytes(npts, r.K, r.cap, o["nobs"]) // 4 + 1, 0)
        m = min(npts, C - 1)                          # its d_ptr (m + 1 entries) fits the verdict-slot buffer
        d_pts, o_obs, o_nobs = _dev(np.arange(m)), _full(o["nobs"]), _full(1)
        o_scr = _full(B.CovisibilityGraph.observations_scratch_bytes(npts, r.K, r.cap, o["nobs"]) // 4 + 1, 0)
        A, Bs = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)
        torch.cuda.synchronize()   # everything allocated and uploaded; from here on only enqueues until the sync
        with torch.cuda.stream(A):
            torch.cuda._sleep(SPIN)
        r.g.observations_device(m, d_pts.data_ptr(), npts, bufs["kf_mp"].data_ptr(), bufs["counts"].data_ptr(), r.K, r.cap, o["nobs"],
                                bufs["vs"].data_ptr(), o_obs.data_ptr(), o_nobs.data_ptr(), o_scr.data_ptr(), stream=A.cuda_stream)
        got, _ = r.device(cur, a=a, obs_cap=o["nobs"], stream=Bs.cuda_stream, bufs=bufs, scr=scr)
        assert got["vs"][:n].tolist() == o["verdict_slot"].tolist() and got["vd"][:n].tolist() == o["verdict"].tolist()
        assert KC.RETIRED in o["verdict"].tolist()
    finally:
        r.close()
