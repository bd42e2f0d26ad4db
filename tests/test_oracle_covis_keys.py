"""CPU test of the covisibility graph and its readers on pointer-sized order keys (tests/covis_key_scenes.py).

Every small scene of tests/covis_scenes.py, observation_scenes.py, kf_culling_scenes.py and local_map_scenes.py runs under
every key map on the reference's own code, its KeyFrames laid out in key order (oracle.covis.RefCovis.set_kf_order), and on
the oracle given the keys; after every step the two agree on everything the existing test_oracle_* files compare (ordered
lists, weights, parents, inputs; observation lists and ref_obs; verdicts, rows, point flags, reference slots; local lists
and the reference keyframe).  Under the monotone maps the oracle's outputs equal those of `small` exactly.  The maps reach
what they are built for: the maximal key in counters and event lists whose sizes are not powers of two, a counter
straddling the low word's wrap, a reference keyframe and a culling order that differ from creation order.  And a numpy
restatement of the device's key sort (cv_sort<false> of orb_slam_b200/csrc/covis.cu) keeps every real entry ahead of the
padding when one key is 2^64 - 1, where the key-only comparison it replaced loses one."""
import numpy as np
import pytest

import covis_key_scenes as KM
import covis_scenes as S
import kf_culling_scenes as KS
import local_map_scenes as LS
import observation_scenes as OS
import test_oracle_covis as TC
import test_oracle_kf_culling as TK
import test_oracle_local_map as TL
import test_oracle_observations as TO
from oracle import covis as OC
from oracle import kf_culling as KC
from oracle import local_map as LM

# a prebuilt oracle/_ref/ older than ref_cv_set_kf_order is only rebuilt where the reference sources are present
needs_ref = pytest.mark.skipif(not (OC.ref_kf_order_available() and KC.ref_kf_order_available() and LM.ref_kf_order_available()),
                               reason="oracle/_ref/ drivers not built with ref_cv_set_kf_order (needs the reference sources)")

FAMILIES = {
    "covis": (S.small_scenes, lambda sc, keys, tr: TC.run(sc, keys=keys, trace=tr)),
    "observations": (OS.small_scenes, lambda sc, keys, tr: TO.run(sc, keys=keys, trace=tr)),
    "kf_culling": (KS.small_scenes, lambda sc, keys, tr: TK.run(sc, keys=keys, trace=tr)),
    "local_map": (LS.small_scenes, lambda sc, keys, tr: TL.run(sc, keys=keys, trace=tr)),
}


def _traces(family, scene):
    """{map: the oracle's outputs after every step}, the reference checked against the oracle under every map"""
    play = FAMILIES[family][1]
    out = {}
    for name in KM.NAMES:
        tr = []
        play(scene, KM.keys(name, scene.nkf), tr)
        out[name] = tr
    return out


_CACHE = {}


def traces(family, name):
    if (family, name) not in _CACHE:
        scene = next(s for s in FAMILIES[family][0]() if s.name == name)
        _CACHE[(family, name)] = _traces(family, scene)
    return _CACHE[(family, name)]


CASES = [(f, s.name) for f, (scenes, _) in FAMILIES.items() for s in scenes()]


@needs_ref
@pytest.mark.parametrize("family,scene", CASES, ids=["%s-%s" % c for c in CASES])
def test_reference_decides_every_key_map(family, scene):
    """the oracle equals the reference after every step under every map (asserted inside the runs); under the monotone
    maps the oracle's outputs are those of `small`, slot for slot"""
    tr = traces(family, scene)
    assert len(tr["small"]) > 0
    for name in KM.MONOTONE:
        assert tr[name] == tr["small"], (family, scene, name)


def _counter(model, k):
    """KeyFrame::UpdateConnections' KFcounter of keyframe k on the model's map: {keyframe: shared observations}"""
    c = {}
    for m in model.kf_mp[k, :model.nfeat[k]].tolist():
        if m < 0 or model.bad[m]:
            continue
        for o in model.obs[m]:
            if o != k:
                c[o] = c.get(o, 0) + 1
    return c


def _filtered(c, key):
    """the targets of the call's AddConnection events: weights >= 15, else the first maximum in key order"""
    th = [o for o, w in c.items() if w >= 15]
    if th:
        return th
    mx = max(c.values())
    return [min((o for o, w in c.items() if w == mx), key=key)]


def _batches(scene, keys, model_cls=S.Model):
    """every update batch of the scene under `keys`: (the entries' counters, {target: the events applied to it, as their
    senders})"""
    model = model_cls(scene, keys)
    for step in scene.steps:
        model.apply(step)
        if step[0] != "update":
            continue
        ks = step[1]
        cs = [_counter(model, k) for k in ks]
        events = {}
        for q, (k, c) in enumerate(zip(ks, cs)):
            if not c:
                continue
            for t in _filtered(c, model.key):
                own = t in ks and cs[ks.index(t)]
                if not own or q > ks.index(t):   # a slot's own call overwrites the events of entries before it
                    events.setdefault(t, []).append(k)
        yield cs, events


def _pow2(n):
    return n > 0 and n & (n - 1) == 0


def test_top_puts_the_maximal_key_where_padding_follows():
    """under `top` the keyframe of key 2^64 - 1 is in a counter of 3 entries, and among the events a touched slot receives
    in one batch, their number not a power of two"""
    sizes, ev = set(), set()
    for sc in S.small_scenes():
        keys = KM.keys("top", sc.nkf)
        top = sc.nkf - 1
        assert int(keys[top]) == KM.MAX
        for cs, events in _batches(sc, keys):
            sizes |= {len(c) for c in cs if top in c}
            ev |= {len(e) for e in events.values() if top in e}
    assert 3 in sizes and any(not _pow2(n) for n in sizes), sizes
    assert any(not _pow2(n) for n in ev), ev


def test_wrap32_counters_straddle_the_wrap():
    """under `wrap32` some counter holds keys on both sides of the low word's wrap"""
    found = False
    for sc in S.small_scenes():
        keys = KM.keys("wrap32", sc.nkf)
        high = lambda k: int(keys[k]) >> 32
        assert len({high(k) for k in range(sc.nkf)}) == (2 if sc.nkf > 1 else 1)
        for cs, _ in _batches(sc, keys):
            found |= any(len({high(k) for k in c}) == 2 for c in cs)
    assert found


@needs_ref
def test_interleaved_changes_the_reference_keyframe_and_a_culling_order():
    """under `interleaved` mpReferenceKF of some frame, and the candidate order of some cull, differ from `small`"""
    ref_diff = any(a["ref_kf"] != b["ref_kf"] for s in LS.small_scenes()
                   for a, b in zip(traces("local_map", s.name)["interleaved"], traces("local_map", s.name)["small"]))
    assert ref_diff
    order_diff = any(a["verdict_slot"] != b["verdict_slot"] for s in KS.small_scenes()
                     for a, b in zip(traces("kf_culling", s.name)["interleaved"], traces("kf_culling", s.name)["small"]))
    assert order_diff


def test_key_maps_are_what_they_say():
    for n in (1, 2, 3, 9, 30, 2000):
        for name in KM.NAMES:
            k = KM.keys(name, n)
            assert len(np.unique(k)) == n
            assert sorted(KM.rank(k).tolist()) == list(range(n))
            if name in KM.MONOTONE:
                assert (np.diff(k.astype(object)) > 0).all() if n > 1 else True, name
        assert int(KM.keys("top", n)[-1]) == KM.MAX
        if n >= 3:
            assert int(KM.keys("top", n)[0]) < 1 << 40 and int(KM.keys("top", n)[n // 2 - 1]) < 1 << 63 <= int(KM.keys("top", n)[-2])
            assert KM.rank(KM.keys("interleaved", n)).tolist() != list(range(n))
            assert {0, KM.MAX} <= {int(x) for x in KM.keys("random", n)}
        assert len({int(x) & 0xFFFFFFFF for x in KM.keys("high_only", n)}) == 1


# ---- the device's key sort (cv_sort<false> of covis.cu) restated: a bitonic network over n2 = pow2ge(n) entries, padding
# after the n real ones, every compare-exchange of the kernel in the kernel's order
INT_MAX = 2 ** 31 - 1


def bitonic(keys, slots, fixed):
    k_arr, s_arr = keys.copy(), slots.copy()
    n2 = len(k_arr)
    i = np.arange(n2)
    k = 2
    while k <= n2:
        j = k >> 1
        while j > 0:
            l = i ^ j
            m = l > i
            a, b = i[m], l[m]
            ka, kb, sa, sb = k_arr[a], k_arr[b], s_arr[a], s_arr[b]
            if fixed:   # (key, slot) ascending
                b_before_a = (kb < ka) | ((kb == ka) & (sb < sa))
                a_before_b = (ka < kb) | ((ka == kb) & (sa < sb))
            else:       # the key alone
                b_before_a, a_before_b = kb < ka, ka < kb
            swap = np.where((a & k) == 0, b_before_a, a_before_b)
            sa_, sb_ = a[swap], b[swap]
            k_arr[sa_], k_arr[sb_] = k_arr[sb_].copy(), k_arr[sa_].copy()
            s_arr[sa_], s_arr[sb_] = s_arr[sb_].copy(), s_arr[sa_].copy()
            j >>= 1
        k <<= 1
    return k_arr, s_arr


def sort_case(n, where, fixed, rng):
    real = rng.permutation(np.unique(rng.integers(0, 1 << 62, size=2 * n + 8, dtype=np.uint64)))[:n]
    at = {"first": 0, "middle": n // 2, "last": n - 1}[where]
    real[at] = np.uint64(KM.MAX)
    n2 = 1 << (n - 1).bit_length()
    keys = np.concatenate([real, np.full(n2 - n, KM.MAX, np.uint64)])
    slots = np.concatenate([np.arange(n, dtype=np.int64), np.full(n2 - n, INT_MAX if fixed else -1, np.int64)])
    k, s = bitonic(keys, slots, fixed)
    want = np.argsort(real, kind="stable")
    return s[:n].tolist() == want.tolist() and k[:n].tolist() == real[want].tolist()


SORT_SIZES = sorted(set(range(1, 71)) | {v for j in range(1, 12) for v in (2 ** j - 1, 2 ** j, 2 ** j + 1) if v <= 2049})


def test_key_sort_keeps_the_maximal_key_ahead_of_padding():
    """with (key, slot) order and padding (2^64 - 1, INT_MAX) the first n entries are the input in key order, the maximal
    key first, in the middle or last; the key-only order with padding (2^64 - 1, -1) loses the real entry in some of them"""
    rng = np.random.default_rng(5)
    lost = []
    for n in SORT_SIZES:
        for where in ("first", "middle", "last"):
            assert sort_case(n, where, True, rng), (n, where)
            if not sort_case(n, where, False, rng):
                lost.append((n, where))
    assert (3, "first") in lost, lost[:10]
    assert all(not _pow2(n) for n, _ in lost)   # no padding, nothing to tie with
