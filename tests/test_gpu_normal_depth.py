"""GPU parity of the batched MapPoint::UpdateNormalAndDepth: orbfe_normal_and_depth_device on observation lists into the frame
store and the host-array orbfe_normal_and_depth, bit for bit (NaN as NaN) against the oracle, which tests/
test_oracle_normal_depth.py pins to the reference's own MapPoint.cc on the same scenes."""
import numpy as np
import pytest

import oracle as O
import orb_slam_b200 as fe
from oracle import normal_depth as N
from orb_slam_b200 import bow as B

import normal_depth_scenes as S

pytestmark = pytest.mark.gpu

SCENES = S.all_scenes()
IDS = [s["name"] for s in SCENES]
PRE_N, PRE_A, PRE_B = np.float32(7.5), np.float32(-3.25), np.float32(-5.5)   # untouched rows keep these


def _torch():
    import torch
    return torch, torch.device("cuda", 0)


def _prefill(n):
    return np.full((n, 3), PRE_N, np.float32), np.full(n, PRE_A, np.float32), np.full(n, PRE_B, np.float32)


def _kps(octs):
    k = np.zeros(len(octs), fe.KP_DTYPE)
    k["octave"] = octs
    return k


def run_device(m, octs, counts, centers, gp, obs, ref, world, scale_factor, sfs, nobs=None, stream=None):
    """One call on a user stream (or `stream`), outputs prefilled; returns (normal, min_dist, max_dist) after the stream
    finished (no matcher sync)."""
    torch, dev = _torch()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    nf = len(counts)
    cap = len(octs) // nf
    n = len(gp) - 1
    pn, pa, pb = _prefill(n)
    d_kps, d_cnt, d_c, d_gp = t(_kps(octs).view(np.uint8)), t(counts), t(centers), t(gp)
    d_obs, d_ref, d_w = t(obs if len(obs) else np.zeros(1, np.int32)), t(ref), t(world)
    d_n, d_a, d_b = t(pn), t(pa), t(pb)
    s = stream or torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()
    B.normal_and_depth_device(m, n, d_kps.data_ptr(), d_cnt.data_ptr(), nf, cap, d_c.data_ptr(), d_gp.data_ptr(), d_obs.data_ptr(),
                              len(obs) if nobs is None else nobs, d_w.data_ptr(), d_ref.data_ptr(), scale_factor, sfs, d_n.data_ptr(),
                              d_a.data_ptr(), d_b.data_ptr(), s.cuda_stream)
    s.synchronize()
    return d_n.cpu().numpy(), d_a.cpu().numpy(), d_b.cpu().numpy()


def oracle_of_store(octs, counts, centers, gp, obs, ref, world, scale_factor, sfs):
    """The oracle on the store's host gather: observer centres by slot, reference centre and octave by the reference slot."""
    cap = len(octs) // len(counts)
    return N.normal_depth(world, centers[ref // cap], octs[ref], gp, centers[obs // cap] if len(obs) else np.zeros((0, 3), np.float32),
                          scale_factor, sfs, *_prefill(len(gp) - 1))


def _same3(x, y):
    return all(S.same(a, b) for a, b in zip(x, y))


@pytest.mark.parametrize("scene", SCENES, ids=IDS)
def test_scenes_both_entries_equal_oracle(gpu_required, scene):
    sf, sfs = scene["scale_factor"], S.scale_table(scene["scale_factor"], scene["nlevels"])
    w, rc, ro, gp, oc, _ = S.host_arrays(scene)
    want = N.normal_depth(w, rc, ro, gp, oc, sf, sfs, *_prefill(len(gp) - 1))
    m = fe.ORBmatcher(0.6, True)
    octs, counts, centers, gp2, obs, ref, world, cap = S.frame_store(scene)
    dev = run_device(m, octs, counts, centers, gp2, obs, ref, world, sf, sfs)
    m.sync()
    host = B.normal_and_depth(m, w, rc, ro, gp, oc, sf, sfs, *_prefill(len(gp) - 1))
    assert _same3(dev, want), scene["name"]
    assert _same3(host, want), scene["name"]
    assert _same3(host, dev)
    bad = [i for i, p in enumerate(scene["points"]) if p["bad"]]
    for i in bad:                                 # a bad map point is an empty group: untouched
        assert (dev[0][i] == PRE_N).all() and dev[1][i] == PRE_A and dev[2][i] == PRE_B
    m.close()


def _seeded_store(seed, nframes=100, cap=2000, npoints=5000, nlevels=8):
    """nframes keyframes of 3/4 cap to cap features (1500-2000 by default), npoints points of 1-1000 observations (mostly 2-40, a tail to 1000), slots
    drawn over the whole store."""
    rng = np.random.default_rng(seed)
    counts = rng.integers(cap * 3 // 4, cap + 1, nframes).astype(np.int32)
    octs = rng.integers(0, nlevels, nframes * cap).astype(np.int32)
    centers = (rng.standard_normal((nframes, 3)) * 5).astype(np.float32)
    sizes = np.where(rng.random(npoints) < 0.97, rng.integers(2, 41, npoints), rng.integers(1, 1001, npoints))
    sizes[:4] = (1, 32, 33, 1000)
    frames = rng.integers(0, nframes, int(sizes.sum()))
    obs = (frames * cap + (rng.random(len(frames)) * counts[frames]).astype(np.int64)).astype(np.int32)
    gp = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    ref = obs[gp[:-1]]                           # the first observation's keyframe
    world = (centers[ref // cap] + rng.standard_normal((npoints, 3)) * 20).astype(np.float32)
    return octs, counts, centers, gp, obs, ref, world


def test_seeded_store_both_entries(gpu_required):
    octs, counts, centers, gp, obs, ref, world = _seeded_store(21)
    sf, sfs = 1.2, S.scale_table(1.2, 8)
    want = oracle_of_store(octs, counts, centers, gp, obs, ref, world, sf, sfs)
    m = fe.ORBmatcher(0.6, True)
    dev = run_device(m, octs, counts, centers, gp, obs, ref, world, sf, sfs)
    m.sync()
    cap = len(octs) // len(counts)
    host = B.normal_and_depth(m, world, centers[ref // cap], octs[ref], gp, centers[obs // cap], sf, sfs, *_prefill(len(gp) - 1))
    assert _same3(dev, want) and _same3(host, want)
    # the same store once more on the matcher's stream: same bits
    assert _same3(run_device(m, octs, counts, centers, gp, obs, ref, world, sf, sfs), want)
    m.sync()
    m.close()


def test_malformed_points_fail_only_themselves(gpu_required):
    """Bad group pointers (negative, decreasing, beyond nobs), an observation slot past its frame's count, in a frame >=
    nframes or negative, a reference slot out of range, reference octaves -1 and nlevels: in one launch with good points.
    The bad points keep their prefilled outputs, the good ones are exact, the sync reports ORBFE_ERR_ARG naming the call,
    and the next call on the same matcher is exact."""
    octs, counts, centers, gp, obs, ref, world = _seeded_store(5, nframes=12, cap=512, npoints=400)
    nf, cap = len(counts), 512
    f = int(np.argmin(counts))
    assert counts[f] < cap
    octs = octs.copy()
    obs, gp, ref = obs.copy(), gp.copy(), ref.copy()
    big = [g for g in range(len(gp) - 1) if gp[g + 1] - gp[g] >= 3][::7]
    bad = set()
    obs[gp[big[0]] + 1] = f * cap + counts[f]; bad.add(big[0])       # feature index == count
    obs[gp[big[1]] + 2] = nf * cap + 3; bad.add(big[1])              # frame == nframes
    obs[gp[big[2]]] = -1; bad.add(big[2])                            # negative slot
    ref[big[3]] = nf * cap; bad.add(big[3])                          # reference slot beyond the store
    ref[big[4]] = f * cap + counts[f]; bad.add(big[4])               # reference feature index == count
    r5, r6 = f * cap + 1, f * cap + 2
    octs[r5], octs[r6] = -1, 8                                       # reference octaves outside [0, 8)
    ref[big[5]], ref[big[6]] = r5, r6
    bad.update((big[5], big[6]))
    bad.update(g for g in range(len(ref)) if ref[g] in (r5, r6))      # any other point referencing those features
    gp[big[7] + 1] = gp[big[7]] - 1; bad.add(big[7])                 # decreasing (the next point starts earlier, still valid)
    gp[big[8] + 1] = -3; bad.update((big[8], big[8] + 1))            # decreasing, and the next one starts below 0
    n = len(gp) - 1
    gp[n] = len(obs) + 4; bad.add(n - 1)                              # the last point ends beyond nobs
    sf, sfs = 1.2, S.scale_table(1.2, 8)
    m = fe.ORBmatcher(0.6, True)
    got = run_device(m, octs, counts, centers, gp, obs, ref, world, sf, sfs)
    with pytest.raises(fe.OrbfeError) as e:
        m.sync()
    assert e.value.code == fe.ORBFE_ERR_ARG and "orbfe_normal_and_depth_device" in str(e.value)
    m.sync()   # the flag is cleared by the report
    for g in range(n):
        if g in bad:
            assert (got[0][g] == PRE_N).all() and got[1][g] == PRE_A and got[2][g] == PRE_B, g
            continue
        b, e_ = int(gp[g]), int(gp[g + 1])
        one = oracle_of_store(octs, counts, centers, np.array([0, e_ - b], np.int32), obs[b:e_], ref[g:g + 1], world[g:g + 1], sf, sfs)
        assert S.same(got[0][g], one[0][0]) and S.same(got[1][g], one[1][0]) and S.same(got[2][g], one[2][0]), g
    # the next call on the same matcher, on well-formed input
    octs2, counts2, centers2, gp2, obs2, ref2, world2 = _seeded_store(6, nframes=12, cap=512, npoints=400)
    again = run_device(m, octs2, counts2, centers2, gp2, obs2, ref2, world2, sf, sfs)
    m.sync()
    assert _same3(again, oracle_of_store(octs2, counts2, centers2, gp2, obs2, ref2, world2, sf, sfs))
    m.close()


def test_empty_groups_untouched(gpu_required):
    """Empty groups (bad map points) between full ones, and a launch of only empty groups: their rows keep what was there,
    whatever their reference slot holds, and nothing is reported."""
    octs, counts, centers, gp, obs, ref, world = _seeded_store(8, nframes=10, cap=256, npoints=50)
    sizes = np.diff(gp)
    sizes[::3] = 0
    keep = np.concatenate([obs[gp[g]:gp[g] + sizes[g]] for g in range(len(sizes))])
    gp2 = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    ref2 = ref.copy()
    ref2[::3] = -7                               # never read for an empty group
    sf, sfs = 1.2, S.scale_table(1.2, 8)
    m = fe.ORBmatcher(0.6, True)
    got = run_device(m, octs, counts, centers, gp2, keep, ref2, world, sf, sfs)
    m.sync()
    ref3 = ref2.copy()
    ref3[::3] = 0
    assert _same3(got, oracle_of_store(octs, counts, centers, gp2, keep, ref3, world, sf, sfs))
    assert (got[0][::3] == PRE_N).all() and (got[1][::3] == PRE_A).all() and (got[2][::3] == PRE_B).all()
    only = run_device(m, octs, counts, centers, np.zeros(6, np.int32), np.zeros(0, np.int32), ref2[:5], world[:5], sf, sfs)
    m.sync()
    assert (only[0] == PRE_N).all() and (only[1] == PRE_A).all() and (only[2] == PRE_B).all()
    m.close()


def test_one_observation_list_serves_both_map_point_calls(gpu_required):
    """ProcessNewKeyFrame's pair: ComputeDistinctiveDescriptors and UpdateNormalAndDepth on one observation list (no
    observation in a bad keyframe), enqueued back to back on one stream, both equal to their oracles."""
    torch, dev = _torch()
    octs, counts, centers, gp, obs, ref, world = _seeded_store(13, nframes=60, cap=1024, npoints=2000)
    nf, cap = len(counts), 1024
    sizes = np.diff(gp)
    sizes = np.minimum(sizes, 150)               # the distinctive kernel is N x N per point: keep to one keyframe's sizes
    obs = np.concatenate([obs[gp[g]:gp[g] + sizes[g]] for g in range(len(sizes))]).astype(np.int32)
    gp = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    rng = np.random.default_rng(13)
    desc = rng.integers(0, 256, (nf * cap, 32), dtype=np.uint8)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    n = len(gp) - 1
    pn, pa, pb = _prefill(n)
    d_desc, d_kps, d_cnt, d_c, d_gp, d_obs = t(desc), t(_kps(octs).view(np.uint8)), t(counts), t(centers), t(gp), t(obs)
    d_ref, d_w, d_n, d_a, d_b = t(ref), t(world), t(pn), t(pa), t(pb)
    d_best = torch.full((n,), -9, dtype=torch.int32, device=dev)
    d_mp = torch.zeros((n, 32), dtype=torch.uint8, device=dev)
    m = fe.ORBmatcher(0.6, True)
    s = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()
    B.distinctive_descriptors_device(m, n, d_desc.data_ptr(), d_cnt.data_ptr(), nf, cap, d_gp.data_ptr(), d_obs.data_ptr(), len(obs),
                                     d_best.data_ptr(), d_mp.data_ptr(), s.cuda_stream)
    sfs = S.scale_table(1.2, 8)
    B.normal_and_depth_device(m, n, d_kps.data_ptr(), d_cnt.data_ptr(), nf, cap, d_c.data_ptr(), d_gp.data_ptr(), d_obs.data_ptr(), len(obs),
                              d_w.data_ptr(), d_ref.data_ptr(), 1.2, sfs, d_n.data_ptr(), d_a.data_ptr(), d_b.data_ptr(), s.cuda_stream)
    s.synchronize()
    m.sync()
    best = O.distinctive_descriptors(desc[obs], gp)
    assert np.array_equal(d_best.cpu().numpy(), best)
    assert np.array_equal(d_mp.cpu().numpy(), desc[obs[gp[:-1] + best]])
    got = (d_n.cpu().numpy(), d_a.cpu().numpy(), d_b.cpu().numpy())
    assert _same3(got, oracle_of_store(octs, counts, centers, gp, obs, ref, world, 1.2, sfs))
    m.close()
