"""GPU tests of the covisibility graph and its readers at the sizes include/orbfe_bow.h accepts, on the scenes of
tests/covis_limit_scenes.py (which tests/test_oracle_covis_limits.py shows reach those sizes): counters of 511 .. 2048
entries, max_connections 1 .. 2048 with C and C + 1 neighbours and full hash tables, max_batch 1000 and 1024 with one target
receiving every entry's event and batches touching more than 1024 slots, erases of 2048-entry maps, lists_device with every
nbest edge over more than 1024 rows, observations at caps 4096, 4097 and 8192, a cull of 2048 candidates and local maps of
more than 1024 counted keyframes.  The device equals the oracle after every step; a batch equals batches of one; every
refusal is ORBFE_ERR_CAPACITY, reported once, with the graph unchanged and parent_out all -1, and the next batch equals the
oracle."""
import numpy as np
import pytest

import orb_slam_b200 as fe

import covis_limit_scenes as L
import test_gpu_covis as G
import test_gpu_kf_culling as GK
import test_gpu_local_map as GL
import test_gpu_observations as GO

pytestmark = pytest.mark.gpu


def nbests(C):
    return (-1, 0, 1, 10, C - 1, C, C + 1)


def oracle_lists(orc, rows, which, nbest):
    """(ptr, list, weights) of lists_device from the oracle (a retired slot a map still names is -1)"""
    cache = {}
    ptr, lst, ws = [0], [], []
    for s in rows.tolist():
        if s not in cache:
            sl, w = orc.ordered(s) if which == 0 else orc.weights(s)
            cache[s] = ([x if orc.live(x) else -1 for x in sl], w)
        sl, w = cache[s]
        if which == 0 and nbest > 0:
            sl, w = sl[:nbest], w[:nbest]
        lst += sl
        ws += w
        ptr.append(len(lst))
    return np.array(ptr, np.int32), np.array(lst, np.int32), np.array(ws, np.int32)


def check_graph(r, where, rows=None, all_nbest=False):
    """every slot's lists (or `rows`) through lists_device equal the oracle's, as arrays"""
    rows = np.arange(r.K, dtype=np.int32) if rows is None else np.asarray(rows, np.int32)
    C = r.g.max_connections
    for which in (0, 1):
        for nb in (nbests(C) if all_nbest else (-1,)):
            got = G.export(r.g, rows.tolist(), which, nb)
            want = oracle_lists(r.orc, rows, which, nb)
            for a, b, name in zip(got, want, ("ptr", "list", "weights")):
                assert np.array_equal(a, b), (where, which, nb, name)


def snapshot(r):
    rows = np.arange(r.K).tolist()
    return [G.export(r.g, rows, which, -1) for which in (0, 1)]


def same(a, b):
    return all(np.array_equal(x, y) for p, q in zip(a, b) for x, y in zip(p, q))


def play(scene, max_batch=64, single=False, check=True):
    r = G.Run(scene, single=single, max_batch=max_batch, keys=scene.keys)
    try:
        for t, step in enumerate(scene.steps):
            r.step(step)
            if check and step[0] != "kf":
                check_graph(r, (scene.name, t, step[0]))
        return r
    except BaseException:
        r.close()
        raise


@pytest.mark.parametrize("scene", L.counter_scenes(), ids=lambda s: s.name)
def test_counter_sizes(gpu_required, scene):
    """counters of 511 .. 2048 entries under max_connections 2048; lists_device with every nbest edge over max_keyframes
    rows drawn with repeats (more than 1024 rows from 1025 entries up)"""
    r = play(scene)
    try:
        rows = np.random.default_rng(1).choice(r.K, size=r.K).astype(np.int32)
        assert len(np.unique(rows)) < r.K
        check_graph(r, (scene.name, "lists"), rows, all_nbest=True)
    finally:
        r.close()


@pytest.mark.parametrize("scene", L.capacity_scenes(), ids=lambda s: s.name)
def test_capacity(gpu_required, scene):
    """C and C + 1 neighbours at C = 1, 1000, 1500, 2048; the full table (17 at C = 6, 4097 at C = 2048); a target map
    filled by an event at C = 2048"""
    r = play(scene, check=scene.nkf < 4000)
    try:
        if scene.refused:
            before = snapshot(r)
            d_par = r.update_device([int(r.slot_of[k]) for k in scene.refused])
            with pytest.raises(fe.OrbfeError) as e:
                r.g.sync()
            assert e.value.code == fe.ORBFE_ERR_CAPACITY
            assert (d_par.cpu().numpy() == -1).all()
            assert same(snapshot(r), before)
            r.g.sync()   # reported once
        r.step(("update", scene.after))
        check_graph(r, (scene.name, "after"), all_nbest=scene.nkf < 4000)
    finally:
        r.close()


BATCH = [(s, mb) for s in L.batch_scenes() for mb in ((s.facts["batch"],) if s.name.startswith("batch_hub") else (1000, 1024))]


@pytest.mark.parametrize("scene,max_batch", BATCH, ids=lambda x: x.name if hasattr(x, "name") else "mb%d" % x)
def test_batches(gpu_required, scene, max_batch):
    """a batch of up to 1024 whose entries all send the hub an event (the hub's own call in the middle of the second), and
    a batch touching more than 1024 slots: equal to the oracle after every step, and to the same updates as batches of one"""
    a = play(scene, max_batch=max_batch)
    b = None
    try:
        b = play(scene, max_batch=max_batch, single=True, check=False)
        assert same(snapshot(a), snapshot(b))
    finally:
        a.close()
        if b is not None:
            b.close()


@pytest.mark.parametrize("scene", L.erase_scenes(), ids=lambda s: s.name)
def test_erase(gpu_required, scene):
    """a hub with 2048 neighbours erased; a leaf of a 2048-entry map erased; a slot a 2048-entry map names stale"""
    r = play(scene)
    try:
        check_graph(r, (scene.name, "lists"), all_nbest=True)
        if "stale" in scene.facts:
            hub = int(r.slot_of[scene.facts["hub"]])
            _, lst, _ = G.export(r.g, [hub], 1, 0)
            assert (lst == -1).sum() == 1   # the stale entry is exported as -1
    finally:
        r.close()


@pytest.mark.parametrize("scene", L.obs_scenes(), ids=lambda s: s.name)
def test_observations(gpu_required, scene):
    """full rows at caps 4096, 4097 and 8192, a point at several cells of one row, lists of more than 1024 entries"""
    r = GO.Run(scene, keys=scene.keys)
    rng = np.random.default_rng(3)
    try:
        for t, step in enumerate(scene.steps):
            r.step(step)
            if step[0] not in ("kf", "update"):
                r.check((scene.name, t, step[0]), rng)
    finally:
        r.close()


def test_cull(gpu_required):
    """a current keyframe whose list holds 2048 candidates at cap 8192: verdicts, rows, points made bad along the list;
    then the graph after the erases"""
    scene = L.scene_cull()
    r = GK._play(scene, check_all=False, keys=scene.keys)
    try:
        check_graph(r, (scene.name, "after the erases"))
    finally:
        r.close()


@pytest.mark.parametrize("scene", L.lm_scenes(), ids=lambda s: s.name)
def test_local_map(gpu_required, scene):
    """1026 and 2049 counted keyframes ranked in tiles of 1024, the maximum tied across tiles; a frame of 8192 cells"""
    GL._play(scene, check_all=False, keys=scene.keys).close()
