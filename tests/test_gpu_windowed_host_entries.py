"""The host-array windowed matchers (orbfe_search_by_projection_frames, orbfe_window_search, orbfe_search_local_points,
orbfe_search_by_projection_kf, orbfe_search_by_projection_f1f2, orbfe_guided_search, orbfe_search_for_initialization) on
the inputs that once sent them to a host replay: pairs of one call with different geometries, views whose grid_inv is not
64/(max-min) and whose scale factors are not a float chain, whole-image windows past the default
candidate scratch, empty frames and query sets, and the largest cap / qcap the fused kernel holds.  Every accepted call
equals the oracle bit for bit; the first refused size returns ORBFE_ERR_UNSUPPORTED with a message."""
import ctypes as C

import numpy as np
import pytest

import oracle as O
import orb_slam_b200 as fe
from orb_slam_b200 import matching as M
from orb_slam_b200.synth import noisy_copies, random_descriptors

pytestmark = pytest.mark.gpu

W, H = 640, 480
FX = FY = 500.0
CX, CY, DEPTH = W / 2.0, H / 2.0, 4.0
DX, DY = 3.0, -2.0          # image motion from frame 1 to frame 2
INT_MAX = 2 ** 31 - 1


def _float_chain(sf, nlevels):
    out = np.empty(nlevels, np.float32)
    fe.lib().orbfe_frame_scale_factors(C.c_float(sf), nlevels, out.ctypes.data_as(C.c_void_p))
    return out


def _scene(n1, n2=None, seed=0, octaves=8):
    """Frame 1 with n1 features; frame 2 with n2 features, the first min(n1, n2) of them noisy copies of a permutation of
    frame 1's, moved by (DX, DY) plus noise."""
    n2 = n1 if n2 is None else n2
    rng = np.random.default_rng(seed)

    def kps(n):
        k = np.zeros(n, fe.KP_DTYPE)
        k["x"], k["y"] = rng.uniform(0, W - 1, n), rng.uniform(0, H - 1, n)
        k["octave"], k["angle"] = rng.integers(0, octaves, n), rng.uniform(0, 360, n)
        k["size"], k["response"], k["class_id"] = 31.0, 1.0, -1
        return k
    k1, d1 = kps(n1), random_descriptors(n1, seed + 1)
    k2, d2 = kps(n2), random_descriptors(n2, seed + 2)
    c = min(n1, n2)
    src = rng.permutation(n1)[:c]
    k2[:c] = k1[src]
    k2["x"][:c] = np.clip(k1["x"][src] + DX + rng.normal(0, 0.7, c), 0, W - 1)
    k2["y"][:c] = np.clip(k1["y"][src] + DY + rng.normal(0, 0.7, c), 0, H - 1)
    k2["angle"][:c] = (k1["angle"][src] + rng.normal(8, 3, c)) % 360
    if c:
        d2[:c] = noisy_copies(d1[src], 0.05, seed + 3)
    return (k1, d1), (k2, d2)


def _views(k, d, geom=None):
    """The library's and the oracle's view of one frame.  geom = (min_x, min_y, max_x, max_y, grid_inv_w, grid_inv_h,
    scale_factors); None = the Frame.cc values of a W x H image with 8 levels of 1.2."""
    nl = 8 if geom is None else len(geom[6])
    v, o = M.FrameView(k, d, W, H, nlevels=nl), O.OracleFrame(k, d, W, H, nlevels=nl)
    if geom is not None:
        for c in (v.c, o.c):
            c.min_x, c.min_y, c.max_x, c.max_y, c.grid_inv_w, c.grid_inv_h = geom[:6]
        v.sf[:] = geom[6]
        o.sf[:] = geom[6]
        O.lib().orb_oracle_frame_grid(C.byref(o.c))   # the oracle's grid from the new geometry
    return v, o


def _world(k):
    w = np.empty((len(k), 3), np.float32)
    w[:, 0] = (k["x"] - np.float32(CX)) / np.float32(FX) * np.float32(DEPTH)
    w[:, 1] = (k["y"] - np.float32(CY)) / np.float32(FY) * np.float32(DEPTH)
    w[:, 2] = DEPTH
    return w


def _tcw(dx=DX, dy=DY):
    T = np.zeros((3, 4), np.float32)
    T[0, 0] = T[1, 1] = T[2, 2] = 1
    T[0, 3], T[1, 3] = dx * DEPTH / FX, dy * DEPTH / FY
    return T


def _launches(m):
    return m.counters()[2]


def _every_entry(m, s1, s2, geom=None, whole=False, seed=0):
    """Every host-array windowed entry on frames s1 -> s2 against the oracle.  whole: windows covering the whole image, so
    every feature of the searched frame is a candidate of every query.  Returns {entry: (nmatches, launches)}."""
    (k1, d1), (k2, d2) = s1, s2
    n1, n2 = len(k1), len(k2)
    v1, o1 = _views(k1, d1, geom)
    v2, o2 = _views(k2, d2, geom)
    rng = np.random.default_rng(seed)
    has = (rng.random(n1) < 0.85).astype(np.uint8)
    outl = (rng.random(n1) < 0.05).astype(np.uint8)
    occ = np.full(n2, -1, np.int32)
    occ[rng.random(n2) < 0.03] = 7
    world = _world(k1)
    proj = np.stack([k1["x"] + np.float32(DX), k1["y"] + np.float32(DY)], axis=1).astype(np.float32)
    lv = k1["octave"].astype(np.int32)
    nnr, ori = m.mfNNratio, m.mbCheckOrientation
    out = {}

    def check(name, got, want):
        n0 = _launches(m)
        n, o = got()
        n_o, o_o = want()
        assert n == n_o and np.array_equal(o, o_o), name
        out[name] = (n, _launches(m) - n0)

    th = 2000.0 if whole else 15.0
    check("search_by_projection_frames",
          lambda: (lambda r: (r[0][0], r[1][0]))(M.search_by_projection_frames(m, [v2], [v1], [has], [outl], [world], [_tcw()], FX, FY,
                                                                                CX, CY, th, cur_mp=[occ])),
          lambda: O.search_by_projection_ff(o2, o1, has, outl, world, _tcw(), FX, FY, CX, CY, th, ori, cur_mp=occ))
    win = 2000 if whole else 30
    check("window_search", lambda: M.window_search(m, v1, v2, has, win, -1, INT_MAX),
          lambda: O.window_search(o1, o2, has, win, -1, INT_MAX, nnratio=nnr, check_orientation=ori))
    prev = np.stack([k1["x"], k1["y"]], axis=1).astype(np.float32)
    check("search_for_initialization", lambda: (lambda r: (r[0], np.concatenate([r[1], r[2].ravel().view(np.int32)])))(
              M.search_for_initialization(m, v1, v2, prev, 2000 if whole else 50)),
          lambda: (lambda r: (r[0], np.concatenate([r[1], r[2].ravel().view(np.int32)])))(
              O.search_for_initialization(o1, o2, prev, 2000 if whole else 50, nnratio=nnr, check_orientation=ori)))
    in_view = (rng.random(n1) < 0.9).astype(np.uint8)
    view_cos = np.where(rng.random(n1) < 0.5, 0.9995, 0.95).astype(np.float32)
    th_lp = 600.0 if whole else 3.0
    check("search_local_points", lambda: M.search_local_points(m, v2, in_view, proj, lv, view_cos, d1, th_lp, f_mp=occ),
          lambda: O.search_local_points(o2, in_view, proj, lv, view_cos, d1, th_lp, nnratio=nnr, f_mp=occ))
    # whole: a huge min_dist predicts level 0 for every point, whose window [-1, 1] holds every octave-0 feature
    min_dist = np.full(n1, 1e6, np.float32) if whole else \
        (DEPTH / np.float32(1.2) ** k1["octave"].astype(np.float32) * rng.uniform(0.8, 1.1, n1)).astype(np.float32)
    check("search_by_projection_kf",
          lambda: M.search_by_projection_kf(m, v2, has, world, min_dist, d1, k1["angle"], _tcw(), FX, FY, CX, CY, th, 100, cur_mp=occ),
          lambda: O.search_by_projection_kf(o2, has, world, min_dist, d1, k1["angle"], _tcw(), FX, FY, CX, CY, th, 100, ori, cur_mp=occ))
    check("search_by_projection_f1f2",
          lambda: M.search_by_projection_f1f2(m, v1, v2, has, world, _tcw(), FX, FY, CX, CY, win, f2_mp=occ),
          lambda: O.search_by_projection_f1f2(o1, o2, has, world, _tcw(), FX, FY, CX, CY, win, nnratio=nnr, f2_mp=occ))
    qr = np.full(n1, 2000.0, np.float32) if whole else (np.float32(6.0) * np.float32(1.2) ** k1["octave"]).astype(np.float32)
    lo, hi = (lv - 1).astype(np.int32), lv
    check("guided_search", lambda: M.guided_search(m, v2, proj[:, 0], proj[:, 1], qr, lo, hi, d1, k1["angle"], 0, 64, 1, slot_owner=occ),
          lambda: O.guided_search(o2, proj[:, 0], proj[:, 1], qr, lo, hi, d1, k1["angle"], 0, nnr, 64, 1, slot_owner=occ))
    return out


def _code(fn, *args, **kw):
    with pytest.raises(fe.OrbfeError) as e:
        fn(*args, **kw)
    return e.value.code, str(e.value)


def test_sbp_frames_pairs_with_different_geometries_in_one_call(gpu_required):
    """Current views of one call with different bounds, nlevels and scale factors: one launch per geometry, pairs in any
    order, a frame's arrays shared by views of two geometries."""
    A = None
    B = (-4.5, -3.25, W + 5.75, H + 2.5, np.float32(64) / np.float32(W + 10.25), np.float32(48) / np.float32(H + 5.75),
         _float_chain(1.25, 10))
    Cg = (2.0, 1.0, W - 1.0, H - 2.0, np.float32(64) / np.float32(W - 3.0), np.float32(48) / np.float32(H - 3.0), _float_chain(1.2, 9))
    scenes = [_scene(900, seed=10 * j) for j in range(3)]
    geoms = [A, B, A, Cg, B]
    pairs = [0, 1, 2, 0, 2]          # scene of each pair: pairs 0 and 3 share frame arrays under geometries A and C
    rng = np.random.default_rng(4)
    curs, lasts, ocur, olast, has, outl, world, occ = [], [], [], [], [], [], [], []
    for g, s in zip(geoms, pairs):
        (k1, d1), (k2, d2) = scenes[s]
        v2, o2 = _views(k2, d2, g)
        v1, o1 = _views(k1, d1, None)
        curs.append(v2), lasts.append(v1), ocur.append(o2), olast.append(o1)
        has.append((rng.random(len(k1)) < 0.9).astype(np.uint8))
        outl.append((rng.random(len(k1)) < 0.05).astype(np.uint8))
        world.append(_world(k1))
        o = np.full(len(k2), -1, np.int32)
        o[rng.random(len(k2)) < 0.03] = 5
        occ.append(o)
    T = [_tcw()] * len(pairs)
    for ori in (True, False):
        m = fe.ORBmatcher(0.9, ori)
        n0 = _launches(m)
        nm, mp = M.search_by_projection_frames(m, curs, lasts, has, outl, world, T, FX, FY, CX, CY, 15.0, cur_mp=occ)
        assert _launches(m) - n0 == 3   # geometries A, B and C
        for j in range(len(pairs)):
            n_o, mp_o = O.search_by_projection_ff(ocur[j], olast[j], has[j], outl[j], world[j], T[j], FX, FY, CX, CY, 15.0, ori,
                                                  cur_mp=occ[j])
            assert nm[j] == n_o and np.array_equal(mp[j], mp_o), (ori, j)
            assert n_o > 300
        m.close()
    # a Last map point whose octave the Current view has no scale factor for
    (k1, d1), (k2, d2) = scenes[0]
    v2, _ = _views(k2[k2["octave"] < 6], d2[k2["octave"] < 6], (0.0, 0.0, float(W), float(H), np.float32(64) / np.float32(W),
                                                               np.float32(48) / np.float32(H), _float_chain(1.2, 6)))
    m = fe.ORBmatcher(0.9, True)
    code, msg = _code(M.search_by_projection_frames, m, [v2], [lasts[0]], [np.ones(len(k1), np.uint8)], [np.zeros(len(k1), np.uint8)],
                      [world[0]], [T[0]], FX, FY, CX, CY, 15.0)
    assert code == fe.ORBFE_ERR_ARG and "octave" in msg
    m.close()


def test_own_grid_and_scale_factors(gpu_required):
    """Views whose grid cell sizes are not 64/(max-min), 48/(max-min), with the extractor's scale-factor table and with a
    table of double-precision powers that is not a float chain: every entry reads the view's own values."""
    ex = fe.ORBextractor(1000, 1.2, 8)
    tables = [ex.tables()[0], np.float32(np.float64(1.2) ** np.arange(8))]
    ex.close()
    assert not np.array_equal(tables[1], _float_chain(1.2, 8))
    m = fe.ORBmatcher(0.8, True)
    for sf in tables:
        geom = (0.0, 0.0, float(W), float(H), np.float32(64) / np.float32(W + 7), np.float32(48) / np.float32(H + 5), sf)
        for name, (n, launches) in _every_entry(m, *_scene(1200, seed=3), geom=geom).items():
            assert n > 50 and launches == 1, (name, n, launches)
    m.close()


def test_whole_image_windows_past_the_default_scratch(gpu_required):
    """Every feature a candidate of every query: 400 x ~350 entries per call, past 64 * cap (projection and guided
    entries) and 256 * cap (SearchForInitialization).  Each call relaunches once with the scratch it needs, and the next
    calls on the same matcher equal the oracle."""
    m = fe.ORBmatcher(0.8, True)
    res = _every_entry(m, *_scene(400, seed=7, octaves=1), whole=True)
    for name, (n, launches) in res.items():
        assert launches == 2, (name, launches)
    for name, (n, launches) in _every_entry(m, *_scene(1000, seed=8)).items():
        assert n > 50 and launches == 1, (name, n, launches)
    m.close()


@pytest.mark.parametrize("n1,n2", [(0, 500), (500, 0), (0, 0)])
def test_empty_frames_and_query_sets(gpu_required, n1, n2):
    """An empty query frame gives no queries, an empty searched frame no candidates: zero matches, outputs as the reference
    leaves them."""
    m = fe.ORBmatcher(0.8, True)
    for name, (n, launches) in _every_entry(m, *_scene(n1, n2, seed=11)).items():
        assert n == 0, name
    m.close()


def _unsupported(fn, *args, **kw):
    code, msg = _code(fn, *args, **kw)
    assert code == fe.ORBFE_ERR_UNSUPPORTED and "220 KB" in msg, msg


def test_largest_accepted_cap_and_qcap(gpu_required):
    """sbp_smem_fixed_bytes(cap, qcap) + 16 KB <= 220 KB: 8283 features per frame for SearchByProjection(Frame,Frame) and
    SearchForInitialization, 24826 queries in a 2000-feature frame for the guided entries; one more is refused."""
    m = fe.ORBmatcher(0.9, True)
    for n in (8283, 8284):
        (k1, d1), (k2, d2) = _scene(n, seed=n)
        v1, o1 = _views(k1, d1)
        v2, o2 = _views(k2, d2)
        has, outl, world = np.ones(n, np.uint8), np.zeros(n, np.uint8), _world(k1)
        prev = np.stack([k1["x"], k1["y"]], axis=1).astype(np.float32)
        args = (m, [v2], [v1], [has], [outl], [world], [_tcw()], FX, FY, CX, CY, 15.0)
        if n == 8284:
            _unsupported(M.search_by_projection_frames, *args)
            _unsupported(M.search_for_initialization, m, v1, v2, prev, 50)
            continue
        nm, mp = M.search_by_projection_frames(*args)
        n_o, mp_o = O.search_by_projection_ff(o2, o1, has, outl, world, _tcw(), FX, FY, CX, CY, 15.0, True)
        assert nm[0] == n_o > 1000 and np.array_equal(mp[0], mp_o)
        r = M.search_for_initialization(m, v1, v2, prev, 50)
        r_o = O.search_for_initialization(o1, o2, prev, 50, nnratio=0.9, check_orientation=True)
        assert r[0] == r_o[0] > 100 and np.array_equal(r[1], r_o[1]) and np.array_equal(r[2], r_o[2])
    (k1, d1), (k2, d2) = _scene(24827, 2000, seed=5)
    v2, o2 = _views(k2, d2)
    qu, qv = k1["x"] + np.float32(DX), k1["y"] + np.float32(DY)
    qr = np.full(len(k1), 4.0, np.float32)
    lo, hi = np.full(len(k1), -1, np.int32), np.full(len(k1), -1, np.int32)
    _unsupported(M.guided_search, m, v2, qu, qv, qr, lo, hi, d1, k1["angle"], 1, 0, 1)
    q = slice(0, 24826)
    n, so = M.guided_search(m, v2, qu[q], qv[q], qr[q], lo[q], hi[q], d1[q], k1["angle"][q], 1, 0, 1)
    n_o, so_o = O.guided_search(o2, qu[q], qv[q], qr[q], lo[q], hi[q], d1[q], k1["angle"][q], 1, 0.9, 0, 1)
    assert n == n_o > 500 and np.array_equal(so, so_o)
    m.close()
