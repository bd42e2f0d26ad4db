"""GPU tests of orbfe_vocabulary_load_text (include/orbfe_bow.h): the table parsed on the device equals the reference's
m_nodes after loadFromTextFile (oracle/voc_text.py), field for field and every weight bit for bit, on synthetic trees, the
head of the real ORBvoc.txt (tests/golden/orbvoc_head.txt) and crafted texts; every rejection names its line; and a loaded
vocabulary drives transform and the device BoW chain exactly as the reference and the same table built with
orbfe_vocabulary_create do.  The reference is given each text without its final newline (see oracle/voc_text.py)."""
import os

import numpy as np
import pytest

import orb_slam_b200 as fe
from orb_slam_b200 import bow as B
from orb_slam_b200.synth import random_vocabulary, noisy_copies, random_descriptors
from oracle import ref as R
from oracle import voc_text as VT

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "orbvoc_head.txt")
KEYS = ("node_desc", "child_ptr", "children", "word_id", "parent")


def ref_nodes(path, tmp_path):
    ref = VT.RefVocabularyNodes(VT.text_for_reference(path, str(tmp_path / ("ref_" + os.path.basename(path)))))
    try:
        return ref.info(), ref.nodes()
    finally:
        ref.close()


def check_against_reference(path, tmp_path):
    info, want = ref_nodes(path, tmp_path)
    V = B.Vocabulary.load_text(path)
    try:
        got, ginfo = V.export(), V.info()
    finally:
        V.close()
    assert ginfo == {"k": info["k"], "L": info["L"], "scoring": info["scoring"], "weighting": info["weighting"],
                     "nnodes": info["nnodes"], "nwords": max(info["nwords"], 1)}
    for k in KEYS:
        assert np.array_equal(got[k], want[k]), k
    assert np.array_equal(got["weight"].view(np.uint64), want["weight"].view(np.uint64))
    return got


def write_text(voc, path, fmt, scoring=0, weighting=0, newline=True):
    """The text of a synthetic vocabulary with weights printed by `fmt` (%r: shortest round trip, mostly 16-17 digits)."""
    nd, cp, ch = voc["node_desc"], voc["child_ptr"], voc["children"]
    n = len(nd)
    parent = np.zeros(n, np.int64)
    parent[ch] = np.repeat(np.arange(n), np.diff(cp))
    leaf = (np.diff(cp) == 0).astype(int)
    desc = [" ".join(map(str, row)) for row in nd.tolist()]
    w = voc["weight"].tolist()
    lines = ["%d %d %d %d" % (voc["k"], voc["L"], scoring, weighting)]
    lines += ["%d %d %s  %s" % (parent[i], leaf[i], desc[i], fmt % w[i]) for i in range(1, n)]
    with open(path, "w") as f:
        f.write("\n".join(lines) + ("\n" if newline else ""))
    return path


@pytest.fixture(scope="module")
def orbvoc_shaped(tmp_path_factory):
    """k = 10, L = 6: the 1,111,111 nodes of ORBvoc.txt, weights printed with %r (nearly all on the host path)."""
    voc = random_vocabulary(10, 6, seed=5)
    path = str(tmp_path_factory.mktemp("vt") / "k10L6.txt")
    return voc, write_text(voc, path, "%r")


def test_orbvoc_shape_equals_reference(gpu_required, orbvoc_shaped, tmp_path):
    voc, path = orbvoc_shaped
    got = check_against_reference(path, tmp_path)
    assert len(got["word_id"]) == 1111111
    assert np.array_equal(got["children"], voc["children"]) and np.array_equal(got["weight"], voc["weight"])


def test_same_file_twice_gives_identical_tables(gpu_required, orbvoc_shaped):
    _, path = orbvoc_shaped
    a, b = B.Vocabulary.load_text(path), B.Vocabulary.load_text(path)
    try:
        ea, eb = a.export(), b.export()
    finally:
        a.close()
        b.close()
    for k in KEYS:
        assert np.array_equal(ea[k], eb[k]), k
    assert np.array_equal(ea["weight"].view(np.uint64), eb["weight"].view(np.uint64))


@pytest.mark.parametrize("k, L, seed, ragged", [(10, 2, 0, False), (4, 5, 1, True), (3, 8, 2, True), (20, 3, 3, False)])
@pytest.mark.parametrize("fmt", ["%r", "%.6g"], ids=["repr", "6digits"])
@pytest.mark.parametrize("newline", [True, False], ids=["newline", "no_newline"])
def test_synthetic_shapes_equal_reference(gpu_required, tmp_path, k, L, seed, ragged, fmt, newline):
    voc = random_vocabulary(k, L, seed=seed, ragged=ragged)
    check_against_reference(write_text(voc, str(tmp_path / "v.txt"), fmt, scoring=seed % 6, weighting=seed % 4, newline=newline),
                            tmp_path)


def test_golden_orbvoc_head_equals_reference(gpu_required, tmp_path):
    got = check_against_reference(GOLDEN, tmp_path)
    assert len(got["word_id"]) == 1112
    # internal nodes whose children the prefix cut off are leaves with word id 0
    assert (np.diff(got["child_ptr"]) == 0).sum() > (got["word_id"] > 0).sum()


def _desc(rng, lo=0, hi=256):
    return [str(int(x)) for x in rng.integers(lo, hi, 32)]


def _crafted(tmp_path, name, body_lines, header="10 6 0 0", eol="\n", final=True):
    p = str(tmp_path / name)
    with open(p, "w", newline="") as f:
        f.write(eol.join([header] + body_lines) + (eol if final else ""))
    return p


WEIGHT_TOKENS = ["1.5", "+1.5", ".5", "5.", "-0", "0", "1E+2", "1e-05", "0.000123456789012345", "1.2345678901234567",
                 "12345678901234567890", "1e-300", "1e400", "inf", "nan", "-inf", "0x1p3", "", "1.5abc", "+", ".", "1e",
                 "4.9e-324", "123456789012345678901234567890.5", "7 trailing tokens ignored", "2.5e22", "3e-22", "999999999999999"]


def test_crafted_weights_and_tokens(gpu_required, tmp_path):
    rng = np.random.default_rng(0)
    lines = ["0 1 %s %s" % (" ".join(_desc(rng)), w) for w in WEIGHT_TOKENS]
    check_against_reference(_crafted(tmp_path, "w.txt", lines), tmp_path)


@pytest.mark.parametrize("eol, sep", [("\r\n", " "), ("\n", "\t"), ("\n", "  \t "), ("\r\n", "\t\r")],
                         ids=["crlf", "tabs", "mixed", "crlf_tabs"])
@pytest.mark.parametrize("final", [True, False], ids=["newline", "no_newline"])
def test_crafted_whitespace(gpu_required, tmp_path, eol, sep, final):
    rng = np.random.default_rng(1)
    lines = []
    for nid in range(1, 300):
        toks = [str(int(rng.integers(0, nid))), str(int(rng.integers(-1, 3)))] + _desc(rng) + ["%.4f" % rng.uniform(0, 9)]
        lines.append(sep.join(toks) + (sep if nid % 7 == 0 else ""))
    check_against_reference(_crafted(tmp_path, "ws.txt", lines, header=sep.join("10 6 0 0".split()), eol=eol, final=final), tmp_path)


def test_crafted_flags_bytes_and_interleaved_siblings(gpu_required, tmp_path):
    """isLeaf of 2 and -1, leaf-flagged nodes that later get children, descriptor values 256, -1 and beyond, signs and leading
    zeros, and parents drawn at random from every earlier node, so siblings are interleaved across the file."""
    rng = np.random.default_rng(2)
    lines = []
    for nid in range(1, 50001):
        pid = int(rng.integers(0, nid)) if nid > 1 else 0
        leaf = ["0", "1", "2", "-1", "+1", "007"][int(rng.integers(0, 6))]
        desc = _desc(rng, -300, 600)
        desc[int(rng.integers(0, 32))] = ["256", "-1", "+5", "-0", "0255"][nid % 5]
        w = ["%.6g" % rng.uniform(0, 9), repr(float(rng.uniform(0, 9))), "0"][nid % 3]
        lines.append("%d %s %s %s" % (pid, leaf, " ".join(desc), w))
    got = check_against_reference(_crafted(tmp_path, "flags.txt", lines), tmp_path)
    assert (np.diff(got["child_ptr"]) > 1).sum() > 1000


def test_parent_with_100k_children(gpu_required, tmp_path):
    rng = np.random.default_rng(3)
    lines, nid = [], 1
    for _ in range(100000 + 3000):
        pid = 0 if rng.random() < 100000 / 103000 or nid < 3 else int(rng.integers(1, nid))
        lines.append("%d 1 %s %.5f" % (pid, " ".join(_desc(rng)), rng.uniform(0, 9)))
        nid += 1
    got = check_against_reference(_crafted(tmp_path, "wide.txt", lines), tmp_path)
    assert got["child_ptr"][1] > 99000


@pytest.mark.parametrize("text", ["10 6 0 0", "10 6 0 0\n", "10 6 0 0\r\n", "3 2 1 2 extra tokens\n"],
                         ids=["bare", "newline", "crlf", "extra"])
def test_header_only(gpu_required, tmp_path, text):
    p = str(tmp_path / "h.txt")
    open(p, "w", newline="").write(text)
    got = check_against_reference(p, tmp_path)
    assert len(got["word_id"]) == 1 and len(got["children"]) == 0


# ---- rejections: ORBFE_ERR_ARG naming the first bad line -----------------------------------------------------------------
GOOD = "0 1 " + " ".join(["3"] * 32) + " 1.5"
BAD_LINES = [
    ("", "empty or blank"), ("  \t \r", "empty or blank"),
    ("0 1 " + " ".join(["3"] * 31), "fewer than 34"), ("0", "fewer than 34"),
    ("x 1 " + " ".join(["3"] * 32) + " 1", "parent is not"), ("1.0 1 " + " ".join(["3"] * 32) + " 1", "parent is not"),
    ("0 1.5 " + " ".join(["3"] * 32) + " 1", "isLeaf"), ("0 one " + " ".join(["3"] * 32) + " 1", "isLeaf"),
    ("0 1 12a " + " ".join(["3"] * 31) + " 1", "descriptor"), ("0 1 99999999999 " + " ".join(["3"] * 31) + " 1", "descriptor"),
    ("-1 1 " + " ".join(["3"] * 32) + " 1", "parent is negative"), ("3 1 " + " ".join(["3"] * 32) + " 1", "parent is negative"),
    ("4 1 " + " ".join(["3"] * 32) + " 1", "parent is negative"),
]


@pytest.mark.parametrize("bad, what", BAD_LINES)
def test_rejections_name_the_line(gpu_required, tmp_path, bad, what):
    p = _crafted(tmp_path, "bad.txt", [GOOD, GOOD, bad, GOOD, bad, GOOD])      # node 3 is file line 4
    with pytest.raises(fe.OrbfeError) as e:
        B.Vocabulary.load_text(p)
    assert e.value.code == fe.ORBFE_ERR_ARG
    assert "line 4:" in str(e.value) and what in str(e.value), str(e.value)


def test_blank_line_before_a_final_newline_is_rejected(gpu_required, tmp_path):
    p = _crafted(tmp_path, "nn.txt", [GOOD, GOOD], eol="\n")
    open(p, "a").write("\n")                                                       # "...\n\n": file line 4 is empty
    with pytest.raises(fe.OrbfeError) as e:
        B.Vocabulary.load_text(p)
    assert e.value.code == fe.ORBFE_ERR_ARG and "line 4:" in str(e.value)


def test_loaded_vocabulary_after_rejection_still_loads(gpu_required, tmp_path):
    """A rejected text leaves nothing behind: the next load on the same device works."""
    with pytest.raises(fe.OrbfeError):
        B.Vocabulary.load_text(_crafted(tmp_path, "bad.txt", [GOOD, "", GOOD]))
    V = B.Vocabulary.load_text(_crafted(tmp_path, "good.txt", [GOOD, GOOD]))
    assert V.info()["nnodes"] == 3
    V.close()


# ---- a loaded vocabulary in use -------------------------------------------------------------------------------------------
def _torch():
    import torch
    return torch, torch.device("cuda", 0)


def _chain(V, desc, F, cap, levelsup=4):
    """descend_device -> bow_vector_device / feature_vector_device -> kfdb_add_device (frames 0..F-2) -> kfdb_detect_device
    (relocalisation and loop queries with frame F-1's padded row); every output as host arrays."""
    torch, dev = _torch()
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dt)).to(dev)
    z = lambda n, dt: torch.full((n,), -7, dtype=dt, device=dev)
    d_desc, d_cnt = t(desc, np.uint8), t(np.full(F, cap), np.int32)
    d_leaf, d_node = z(F * cap, torch.int32), z(F * cap, torch.int32)
    d_ids, d_vals, d_n = z(F * cap, torch.int32), z(F * cap, torch.float64), z(F, torch.int32)
    d_fid, d_fptr, d_fit, d_fn = z(F * cap, torch.int32), z(F * (cap + 1), torch.int32), z(F * cap, torch.int32), z(F, torch.int32)
    torch.cuda.synchronize()
    V.descend_device(d_desc.data_ptr(), F * cap, levelsup, d_leaf.data_ptr(), d_node.data_ptr())
    B.bow_vector_device(V, F, d_leaf.data_ptr(), d_cnt.data_ptr(), cap, d_ids.data_ptr(), d_vals.data_ptr(), d_n.data_ptr())
    B.feature_vector_device(V, F, d_leaf.data_ptr(), d_node.data_ptr(), d_cnt.data_ptr(), cap, d_fid.data_ptr(), d_fptr.data_ptr(),
                            d_fit.data_ptr(), d_fn.data_ptr())
    db = B.KeyFrameDatabase(V, F, F * cap)
    db.add_device(np.arange(F - 1), np.arange(F - 1), cap, d_ids.data_ptr(), d_vals.data_ptr(), d_n.data_ptr())
    out = {k: x.cpu().numpy() for k, x in (("leaf", d_leaf), ("node", d_node), ("bow_ids", d_ids), ("bow_vals", d_vals),
                                           ("bow_n", d_n), ("fv_ids", d_fid), ("fv_ptr", d_fptr), ("fv_items", d_fit), ("fv_n", d_fn))}
    q = (F - 1) * cap
    for mode in (db.RELOC, db.LOOP):
        d_cand, d_nc, d_w, d_s = z(F, torch.int32), z(1, torch.int32), z(F, torch.int32), z(F, torch.float32)
        torch.cuda.synchronize()
        db.detect_device(mode, cap, d_ids[q:].data_ptr(), d_vals[q:].data_ptr(), 0, 0, 0.01, F, d_cand.data_ptr(), d_nc.data_ptr(),
                         d_w.data_ptr(), d_s.data_ptr())
        torch.cuda.synchronize()
        out.update({"cand%d" % mode: d_cand.cpu().numpy(), "ncand%d" % mode: d_nc.cpu().numpy(), "words%d" % mode: d_w.cpu().numpy(),
                    "score%d" % mode: d_s.cpu().numpy()})
    db.close()
    return out


@pytest.mark.parametrize("scoring, weighting", [(0, 0), (1, 2), (5, 1)])
def test_loaded_vocabulary_drives_transform_and_the_device_chain(gpu_required, tmp_path, scoring, weighting):
    voc = random_vocabulary(10, 4, seed=7, ragged=True)
    path = write_text(voc, str(tmp_path / "v.txt"), "%r", scoring=scoring, weighting=weighting)
    loaded = B.Vocabulary.load_text(path)
    table = loaded.export()
    norm = {0: B.NORM_L1, 1: B.NORM_L2, 5: B.NORM_NONE}[scoring]
    created = B.Vocabulary(dict(table, L=4), weighting=weighting, norm=norm)
    assert created.info() == dict(loaded.info(), k=-1, scoring=-1)
    ref = R.RefVocabulary(VT.text_for_reference(path, str(tmp_path / "ref.txt")))
    words = voc["node_desc"][voc["word_id"] >= 0]
    F, cap = 6, 1500
    desc = np.concatenate([noisy_copies(words[np.random.default_rng(f).integers(0, len(words), cap)], 0.08, f) for f in range(F)])
    desc[::37] = random_descriptors(len(desc[::37]), 11)
    desc[(F - 1) * cap:] = noisy_copies(desc[:cap], 0.03, 12)                    # the query revisits frame 0
    try:
        for f in (0, F - 1):
            d = desc[f * cap:(f + 1) * cap]
            (bi, bv), (fi, fp, ff) = loaded.transform(d)
            (rbi, rbv), (rfi, rfp, rff) = ref.transform(d)
            assert np.array_equal(bi, rbi) and np.array_equal(bv.view(np.uint64), rbv.view(np.uint64))
            assert np.array_equal(fi, rfi) and np.array_equal(fp, rfp) and np.array_equal(ff, rff)
        a, b = _chain(loaded, desc, F, cap), _chain(created, desc, F, cap)
        for k in a:
            assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), k
        assert a["ncand1"][0] > 0
    finally:
        loaded.close()
        created.close()
