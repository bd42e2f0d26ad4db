"""The projecting matchers at their rounding edges on the device, match for match against the oracle (which
test_oracle_projection_domain.py holds to the restatement and to the reference's own ORBmatcher): the scenes of
projection_domain_scenes.py through orbfe_search_by_projection_device (every SearchByProjection(Frame, Frame) scene of a scale
in one launch, each pair with its own general Tcw; entries in shared memory and in the global scratch; both
check_orientation values), orbfe_search_by_projection_frames, _f1f2, _kf, orbfe_search_local_points and
orbfe_search_for_triangulation(_device); then one chain extract -> back-project -> orbfe_search_by_projection_device over
consecutive frames of a rotating camera."""
import ctypes as C

import numpy as np
import pytest

import oracle as O
import orb_slam_b200 as fe
import projection_domain_scenes as S
from orb_slam_b200 import matching as M
from orb_slam_b200.synth import textured_frame
from test_oracle_projection_domain import one_node, run_oracle

pytestmark = pytest.mark.gpu

SCENES = S.scenes()


def of(routine):
    return [s for s in SCENES if s.routine == routine]


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(torch.device("cuda", 0))


def view(kps, desc, s):
    return M.FrameView(kps, desc, S.W, S.H, s.scale, s.nlevels)


@pytest.mark.parametrize("scratch", [False, True], ids=["smem", "scratch"])
@pytest.mark.parametrize("ori", [False, True])
@pytest.mark.parametrize("scale", list(S.SCALES))
def test_search_by_projection_device(gpu_required, monkeypatch, scale, ori, scratch):
    """Every SearchByProjection(Frame, Frame) scene of one scale as one pair of one launch (frame 2j = Current, 2j+1 = Last)"""
    import torch
    if scratch:
        monkeypatch.setenv("ORBFE_SBP_FORCE_SCRATCH", "1")
    sc = [s for s in of("ff") if s.name.endswith(scale)]
    assert len(sc) >= 2 and len({s.th for s in sc}) == 1 and len({s.T.tobytes() for s in sc}) == len(sc)
    P = len(sc)
    cap = max(max(len(s.cur_kps), len(s.last_kps)) for s in sc)
    kps = np.zeros((2 * P, cap), S.KP_DTYPE)
    desc = np.zeros((2 * P, cap, 32), np.uint8)
    world = np.zeros((2 * P, cap, 3), np.float32)
    flags = np.zeros((2 * P, cap), np.uint8)
    counts = np.zeros(2 * P, np.int32)
    for j, s in enumerate(sc):
        nc, nl = len(s.cur_kps), len(s.last_kps)
        kps[2 * j, :nc], desc[2 * j, :nc], counts[2 * j] = s.cur_kps, s.cur_desc, nc
        kps[2 * j + 1, :nl], desc[2 * j + 1, :nl], counts[2 * j + 1] = s.last_kps, s.last_desc, nl
        world[2 * j + 1, :nl], flags[2 * j + 1, :nl] = s.world, 1
    T = np.stack([s.T.reshape(12) for s in sc]).astype(np.float32)
    d_mp, d_nm = dev(np.full((P, cap), -1, np.int32)), torch.full((P,), -9, dtype=torch.int32, device="cuda:0")
    d = [dev(kps.view(np.uint8).reshape(2 * P, cap, 28)), dev(desc), dev(counts), dev(np.arange(0, 2 * P, 2, dtype=np.int32)),
         dev(np.arange(1, 2 * P, 2, dtype=np.int32)), dev(world), dev(flags), dev(T)]
    s0 = sc[0]
    m = fe.ORBmatcher(0.9, ori)
    M.search_by_projection_device(m, P, *[x.data_ptr() for x in d[:3]], cap, *[x.data_ptr() for x in d[3:]], S.W, S.H, s0.scale,
                                  s0.nlevels, float(S.FX), float(S.FY), float(S.CX), float(S.CY), s0.th, d_mp.data_ptr(), d_nm.data_ptr())
    m.sync()
    m.close()
    mp, nm = d_mp.cpu().numpy(), d_nm.cpu().numpy()
    for j, s in enumerate(sc):
        n_o, mp_o = run_oracle(s, ori)
        assert nm[j] == n_o and np.array_equal(mp[j, :len(s.cur_kps)], mp_o), s.name


@pytest.mark.parametrize("s", of("ff"), ids=lambda s: s.name)
def test_search_by_projection_frames(gpu_required, s):
    n = len(s.world)
    m = fe.ORBmatcher(0.9, True)
    nm, mp = M.search_by_projection_frames(m, [view(s.cur_kps, s.cur_desc, s)], [view(s.last_kps, s.last_desc, s)], [np.ones(n, np.uint8)],
                                           [np.zeros(n, np.uint8)], [s.world], [s.T], float(S.FX), float(S.FY), float(S.CX),
                                           float(S.CY), s.th)
    m.close()
    n_o, mp_o = run_oracle(s, True)
    assert nm[0] == n_o and np.array_equal(mp[0], mp_o)


@pytest.mark.parametrize("s", of("f1f2"), ids=lambda s: s.name)
def test_search_by_projection_f1f2(gpu_required, s):
    m = fe.ORBmatcher(s.nnratio, False)
    n, mp = M.search_by_projection_f1f2(m, view(s.f1_kps, s.f1_desc, s), view(s.f2_kps, s.f2_desc, s), np.ones(len(s.world), np.uint8),
                                        s.world, s.T, float(S.FX), float(S.FY), float(S.CX), float(S.CY), s.window)
    m.close()
    n_o, mp_o = run_oracle(s)
    assert n == n_o and np.array_equal(mp, mp_o)


@pytest.mark.parametrize("ori", [False, True])
@pytest.mark.parametrize("s", of("kf"), ids=lambda s: s.name)
def test_search_by_projection_kf(gpu_required, s, ori):
    n = len(s.world)
    m = fe.ORBmatcher(0.9, ori)
    nm, mp = M.search_by_projection_kf(m, view(s.cur_kps, s.cur_desc, s), np.ones(n, np.uint8), s.world, s.min_dist, s.desc,
                                       np.zeros(n, np.float32), s.T, float(S.FX), float(S.FY), float(S.CX), float(S.CY), s.th, s.orb_dist)
    m.close()
    n_o, mp_o = run_oracle(s, ori)
    assert nm == n_o and np.array_equal(mp, mp_o)


@pytest.mark.parametrize("s", of("local"), ids=lambda s: s.name)
def test_search_local_points(gpu_required, s):
    m = fe.ORBmatcher(s.nnratio, False)
    n, mp = M.search_local_points(m, view(s.kps, s.desc, s), np.ones(len(s.proj), np.uint8), s.proj, s.level, s.view_cos, s.mp_desc, s.th)
    m.close()
    n_o, mp_o = run_oracle(s)
    assert n == n_o and np.array_equal(mp, mp_o)


@pytest.mark.parametrize("ori", [False, True])
@pytest.mark.parametrize("s", of("tri"), ids=lambda s: s.name)
def test_search_for_triangulation(gpu_required, s, ori):
    """the host-array entry, and the device entry with the scene as job (0, 1) and again as (1, 0) with F12 transposed
    (the same pairs seen from side 2, against the oracle on that job)"""
    import torch
    n1, n2 = len(s.k1), len(s.k2)
    n_o, m12_o = run_oracle(s, ori)
    m = fe.ORBmatcher(0.6, ori)
    n_h, m12_h = M.search_for_triangulation(m, s.k1, s.d1, np.zeros(n1, np.uint8), one_node(n1), s.k2, s.d2, np.zeros(n2, np.uint8),
                                            one_node(n2), s.F12, s.sig2)
    assert n_h == n_o and np.array_equal(m12_h, m12_o)
    cap = max(n1, n2)
    kps = np.zeros((2, cap), S.KP_DTYPE)
    desc = np.zeros((2, cap, 32), np.uint8)
    kps[0, :n1], desc[0, :n1], kps[1, :n2], desc[1, :n2] = s.k1, s.d1, s.k2, s.d2
    ids, items = np.zeros((2, cap), np.int32), np.zeros((2, cap), np.int32)
    ptr = np.zeros((2, cap + 1), np.int32)
    for f, n in enumerate((n1, n2)):
        ptr[f, 1], items[f, :n] = n, np.arange(n)
    F21 = s.F12.reshape(3, 3).T.copy()
    F = np.stack([s.F12.reshape(9), F21.reshape(9)]).astype(np.float32)
    d = [dev(kps.view(np.uint8).reshape(2, cap, 28)), dev(desc), dev(np.array([n1, n2], np.int32)), dev(ids), dev(ptr), dev(items),
         dev(np.ones(2, np.int32)), dev(np.zeros((2, cap), np.uint8)), dev(np.array([0, 1], np.int32)), dev(np.array([1, 0], np.int32)),
         dev(F)]
    d_out, d_nm = dev(np.full((2, cap), -9, np.int32)), torch.full((2,), -9, dtype=torch.int32, device="cuda:0")
    M.search_for_triangulation_device(m, 2, *[x.data_ptr() for x in d[:3]], cap, *[x.data_ptr() for x in d[3:]], s.sig2,
                                      d_out.data_ptr(), d_nm.data_ptr())
    m.sync()
    m.close()
    out, nm = d_out.cpu().numpy(), d_nm.cpu().numpy()
    assert nm[0] == n_o and np.array_equal(out[0, :n1], m12_o)
    n_r, m21_o = O.search_for_triangulation(s.k2, s.d2, np.zeros(n2, np.uint8), one_node(n2), s.k1, s.d1, np.zeros(n1, np.uint8),
                                            one_node(n1), F21, s.sig2, check_orientation=ori)
    assert nm[1] == n_r and np.array_equal(out[1, :n2], m21_o)


# ---- one chain on a rotating camera ----------------------------------------------------------------------------------------
def test_chain_extract_backproject_sbp_rotating_camera(gpu_required):
    """orbfe_extract_batch_device -> back-projection of frame i's keypoints at depth 4 -> orbfe_search_by_projection_device of
    frame i + 1 against frame i with a general rotation per step (0.3-0.5 degrees about a tilted axis, plus the image shift's
    translation), against the oracle's extract and SearchByProjection."""
    import torch
    W, H, B, NF = S.W, S.H, 5, 1000
    base = textured_frame(W + 24, H + 24, seed=33)
    imgs = np.stack([np.ascontiguousarray(base[2 * i:2 * i + H, 3 * i:3 * i + W]) for i in range(B)])
    ex = fe.ORBextractor(NF, 1.2, 8, fe.FAST_SCORE, 20, device=0)
    cap = NF
    d_img = dev(imgs)
    d_kps = torch.zeros((B, cap, 28), dtype=torch.uint8, device="cuda:0")
    d_desc = torch.zeros((B, cap, 32), dtype=torch.uint8, device="cuda:0")
    d_cnt = torch.zeros(B, dtype=torch.int32, device="cuda:0")
    ex.extract_batch_device(d_img.data_ptr(), W, H, W, W * H, B, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr())
    ex.sync()
    torch.cuda.synchronize()
    p = O.make_params(NF, 1.2, 8, 1, 20)
    okps, odesc = [], []
    for i in range(B):
        rc, k, dd, _ = O.extract(p, imgs[i])
        okps.append(k)
        odesc.append(dd)
    cnt = d_cnt.cpu().numpy()
    kd = d_kps.cpu().numpy().view(S.KP_DTYPE).reshape(B, cap)
    for i in range(B):
        assert cnt[i] == len(okps[i]) and np.array_equal(kd[i, :cnt[i]], okps[i])
    ex.close()
    for n_o in sbp_chain(d_kps, d_desc, d_cnt, cap, okps, odesc, [(i + 1, i) for i in range(B - 1)], W, H):
        assert n_o > 50


def sbp_chain(d_kps, d_desc, d_cnt, cap, okps, odesc, pairs, W, H, cx=S.CX, cy=S.CY):
    """orbfe_search_by_projection_device over `pairs` [(current, last)] of a device frame store whose frames hold the
    oracle's keypoints okps / odesc: the last frame's keypoints back-projected at depth 4, a general rotation per pair
    (0.3-0.5 degrees about a tilted axis, plus the translation of a 3 px, 2 px image shift), image bounds (0, 0, W, H); the
    matches equal the oracle's SearchByProjection.  Returns the oracle's match count of each pair."""
    import torch
    F, P = len(okps), len(pairs)
    world = np.zeros((F, cap, 3), np.float32)
    flags = np.zeros((F, cap), np.uint8)
    for i, k in enumerate(okps):
        world[i, :len(k), 0] = (k["x"] - cx) / S.FX * np.float32(4)
        world[i, :len(k), 1] = (k["y"] - cy) / S.FY * np.float32(4)
        world[i, :len(k), 2] = 4
        flags[i, :len(k)] = 1
    T = np.stack([S.pose((0.2, 0.3 * (-1) ** i, 0.93), 0.3 + 0.05 * i, (-3 * 4 / float(S.FX), -2 * 4 / float(S.FY), 0.01))
                  for i in range(P)]).astype(np.float32)
    d_mp = torch.full((P, cap), -1, dtype=torch.int32, device="cuda:0")
    d_nm = torch.zeros(P, dtype=torch.int32, device="cuda:0")
    d_args = [dev(np.array([c for c, _ in pairs], np.int32)), dev(np.array([l for _, l in pairs], np.int32)), dev(world), dev(flags),
              dev(T.reshape(P, 12))]
    m = fe.ORBmatcher(0.9, True)
    L = M._bind()
    rc = L.orbfe_search_by_projection_device(m.handle, P, C.c_void_p(d_kps.data_ptr()), C.c_void_p(d_desc.data_ptr()),
                                             C.c_void_p(d_cnt.data_ptr()), cap, *[C.c_void_p(x.data_ptr()) for x in d_args],
                                             0.0, 0.0, float(W), float(H), 1.2, 8, float(S.FX), float(S.FY), float(cx), float(cy),
                                             7.0, 1, C.c_void_p(d_mp.data_ptr()), C.c_void_p(d_nm.data_ptr()), None)
    assert rc == 0
    m.sync()
    m.close()
    mp, nm = d_mp.cpu().numpy(), d_nm.cpu().numpy()
    out = []
    for j, (c, l) in enumerate(pairs):
        nl = len(okps[l])
        n_o, mp_o = O.search_by_projection_ff(O.OracleFrame(okps[c], odesc[c], W, H), O.OracleFrame(okps[l], odesc[l], W, H),
                                              np.ones(nl, np.uint8), np.zeros(nl, np.uint8), world[l, :nl], T[j], S.FX, S.FY, cx,
                                              cy, 7.0, check_orientation=True)
        assert nm[j] == n_o and np.array_equal(mp[j, :len(okps[c])], mp_o), (c, l)
        out.append(n_o)
    return out
