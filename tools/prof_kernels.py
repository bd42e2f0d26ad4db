#!/usr/bin/env python3
"""Measurement harness for the configurations that are not the bench line (run on one H100):

  --what config3   BASELINE configs[2]: 3840x2160, 4000 kp, 12 levels -- per-stage CUDA-event times of the extractor on a
                   device-resident batch, achieved GB/s against the 130.86 MB/frame of SURVEY.md 8(d)
  --what config5   BASELINE configs[4]: 2000 query descriptors x (ngroups keyframes x 2000 descriptors): the brute-force
                   best/second sweep (knn2 kernel), Gpairs/s, HBM GB/s, POPC-pipe estimate
  --what small     the latency-bound kernels once each (bow_descend, distinctive, undistort, hamming_csr, sbp single pair,
                   feature_vector, search_by_bow, search_for_triangulation) so that an `ncu -k regex:` capture finds them
  --what reloc     SearchByBoW at its two call sites, device-resident: relocalisation (one 1080p / 2000-keypoint frame against
                   32 candidate keyframes, KeyFrame-vs-Frame overload) and loop closing (one keyframe against 16 candidates,
                   KeyFrame-vs-KeyFrame); CUDA-event ms of the FeatureVector build and of the batched search, next to the wall
                   time of the same jobs one pair per call through the host-array entry orbfe_search_by_bow (staging, one
                   launch and a synchronise per pair)
  --what mapping   SearchForTriangulation at LocalMapping::CreateNewMapPoints: one 1080p / 2000-keypoint keyframe against 20
                   neighbours, F12 from the poses as ComputeF12; CUDA-event ms of the batched call next to the wall time of the
                   same jobs one pair per call through the host-array entry orbfe_search_for_triangulation (staging, one
                   launch and a synchronise per pair), and same_as_host
  --what mapdesc   ComputeDistinctiveDescriptors at LocalMapping::ProcessNewKeyFrame: the 2000 map points of one 2000-feature
                   keyframe over a 60-keyframe store (synthetic descriptors), with and without one 1000-observation point;
                   CUDA-event ms of
                   orbfe_distinctive_descriptors_device next to the wall time of orbfe_distinctive_descriptors including the
                   host gather of the descriptors, and same_as_host
  --what kfdb      the resident KeyFrameDatabase at 1k and 10k keyframes of ~1000 words (ids over 10^6): CUDA-event ms per loop
                   and per relocalisation query, host ms per add / erase, and the wall time of the stateless
                   orbfe_bow_db_detect on the same data
  --what bowchain  the BowVector kernel alone for 1 and 33 1080p / 2000-keypoint frames (CUDA events), relocalisation from an
                   extracted frame to SearchByBoW results against a resident 1000-keyframe database with the BowVector built
                   on the device vs on the host (wall time), and detect_device on a padded row vs its word count
  --what windowed  wall time per call of the host-array windowed matchers (staging, launch, copy back, synchronise):
                   orbfe_search_by_projection_frames for 1 and 8 pairs, orbfe_search_local_points and orbfe_window_search at
                   1080p / 2000 keypoints, orbfe_search_for_initialization at 720p / 2000 keypoints

Prints one JSON object per --what; never a bench value when run under ncu."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def level_sizes(W, H, nlevels, scale=1.2):
    inv = np.float32(np.float32(1.0) / np.float64(np.float32(scale)))
    s = np.float32(1.0)
    out = []
    for _ in range(nlevels):
        out.append((int(np.rint(np.float32(W) * s)), int(np.rint(np.float32(H) * s))))
        s = np.float32(s * inv)
    return out


def config3(args):
    import torch
    import orb_slam_b200 as fe
    from orb_slam_b200.synth import textured_frame, shifted_frame
    W, H, NF, NL = 3840, 2160, 4000, 12
    B = args.batch
    base = textured_frame(W, H, seed=33)
    frames = np.stack([base] + [shifted_frame(base, 3 * i, 2 * i, seed=i) for i in range(1, B)])
    dev = torch.device("cuda", 0)
    d_frames = torch.from_numpy(frames).to(dev)
    d_kps = torch.empty((B, NF, 28), dtype=torch.uint8, device=dev)
    d_desc = torch.empty((B, NF, 32), dtype=torch.uint8, device=dev)
    d_cnt = torch.empty((B,), dtype=torch.int32, device=dev)
    ex = fe.ORBextractor(NF, 1.2, NL, fe.FAST_SCORE, 20)
    stream = torch.cuda.Stream(device=dev)
    ex.set_profiling(True)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def run(n):
        for _ in range(n):
            ex.extract_batch_device(d_frames.data_ptr(), W, H, W, W * H, B, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(),
                                    stream.cuda_stream)
    run(args.warmup)
    stream.synchronize()
    ex.stage_times()
    with torch.cuda.stream(stream):
        e0.record(stream)
        run(args.iters)
        e1.record(stream)
    stream.synchronize()
    total_ms = e0.elapsed_time(e1) / args.iters
    acc = {}
    for name, ms in ex.stage_times():
        acc[name] = acc.get(name, 0.0) + ms / args.iters
    ls = level_sizes(W, H, NL)
    P = sum(w * h for w, h in ls)
    reads = sum(w * h for w, h in ls[:-1]) + 2 * P
    writes = (P - W * H) + P
    alg = reads + writes + NF * (749 + 512) + NF * 60
    peak = 3350.0   # H100 SXM data sheet; MEASURED_PEAKS.json replaces it where the machine provides one
    try:
        peak = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        pass
    kern_ms = sum(v for k, v in acc.items() if k != "ingest")
    out = {"what": "config3: 3840x2160, 4000 kp, 12 levels, batch %d device-resident" % B, "counts": d_cnt.cpu().numpy().tolist(),
           "ms_per_batch": total_ms, "ms_per_frame": total_ms / B, "stage_ms_per_batch": acc,
           "algorithmic_MB_per_frame": alg / 1e6, "P_px": P,
           "extract_kernels": {"ms_per_batch": kern_ms, "achieved_GBs": alg * B / (kern_ms * 1e-3) / 1e9,
                               "frac_of_measured_hbm_peak": alg * B / (kern_ms * 1e-3) / 1e9 / peak},
           "fast_nms": {"achieved_GBs": P * B / (acc.get("fast_nms", 1e9) * 1e-3) / 1e9,
                        "frac_of_measured_hbm_peak": P * B / (acc.get("fast_nms", 1e9) * 1e-3) / 1e9 / peak},
           "pyramid": {"achieved_GBs": (sum(w * h for w, h in ls[:-1]) + P - W * H) * B / (acc.get("pyramid", 1e9) * 1e-3) / 1e9},
           "Mkp_per_s": NF * B / (total_ms * 1e-3) / 1e6, "hbm_peak_GBs": peak}
    ex.close()
    return out


def config5(args):
    import torch
    import orb_slam_b200 as fe
    from orb_slam_b200.synth import random_descriptors
    nq, per, ng = 2000, 2000, args.groups
    dev = torch.device("cuda", 0)
    q = torch.from_numpy(random_descriptors(nq, 1)).to(dev)
    g = torch.Generator(device=dev); g.manual_seed(5)
    db = torch.randint(0, 256, (ng * per, 32), dtype=torch.uint8, device=dev, generator=g)
    best = torch.empty((ng, nq), dtype=torch.uint16, device=dev)
    idx = torch.empty((ng, nq), dtype=torch.int32, device=dev)
    second = torch.empty((ng, nq), dtype=torch.uint16, device=dev)
    m = fe.ORBmatcher()
    L = fe.lib()
    stream = torch.cuda.Stream(device=dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def run(n):
        for _ in range(n):
            rc = L.orbfe_knn2_groups_device(m.handle, C.c_void_p(q.data_ptr()), nq, C.c_void_p(db.data_ptr()), ng, per,
                                            C.c_void_p(best.data_ptr()), C.c_void_p(idx.data_ptr()), C.c_void_p(second.data_ptr()),
                                            C.c_void_p(stream.cuda_stream))
            assert rc == 0, L.orbfe_last_error()
    run(args.warmup)
    stream.synchronize()
    with torch.cuda.stream(stream):
        e0.record(stream)
        run(args.iters)
        e1.record(stream)
    stream.synchronize()
    ms = e0.elapsed_time(e1) / args.iters
    pairs = float(nq) * ng * per
    # spot check against the oracle on one group (outside the timed region)
    chk = None
    try:
        import oracle as O
        gsel = ng // 2
        bd, bi, sd = O.knn2(q.cpu().numpy(), db[gsel * per:(gsel + 1) * per].cpu().numpy())
        chk = bool(np.array_equal(best[gsel].cpu().numpy(), bd) and np.array_equal(idx[gsel].cpu().numpy(), bi)
                   and np.array_equal(second[gsel].cpu().numpy(), np.minimum(sd, 65535)))
    except Exception as e:
        chk = "oracle unavailable: %r" % e
    out = {"what": "config5: %d queries x %d keyframes x %d descriptors, 256-bit Hamming best/second per keyframe" % (nq, ng, per),
           "ms_per_query_set": ms, "Gpairs_per_s": pairs / (ms * 1e-3) / 1e9, "db_MB": ng * per * 32 / 1e6,
           "hbm_GBs": (ng * per * 32 + ng * nq * 8) / (ms * 1e-3) / 1e9,
           "word_ops_per_s_T": pairs * 8 / (ms * 1e-3) / 1e12, "oracle_spot_check": chk}
    m.close()
    return out


def small(args):
    """One call of every latency-bound kernel (for `ncu -k`), sizes of the reference's usage."""
    import torch
    import orb_slam_b200 as fe
    from orb_slam_b200 import matching as M, bow as BW
    from orb_slam_b200.synth import textured_frame, shifted_frame, random_vocabulary, random_descriptors
    W, H = 1920, 1080
    f0 = textured_frame(W, H, seed=9)
    f1 = shifted_frame(f0, 5, -3, seed=1)
    ex = fe.ORBextractor(2000, 1.2, 8)
    (k0, d0), (k1, d1) = ex(f0), ex(f1)
    m = fe.ORBmatcher(0.9, True)
    v0, v1 = M.FrameView(k0, d0, W, H), M.FrameView(k1, d1, W, H)
    world = np.empty((len(k0), 3), np.float32)
    world[:, 0] = (k0["x"] - 960.0) / 1000.0 * 5.0; world[:, 1] = (k0["y"] - 540.0) / 1000.0 * 5.0; world[:, 2] = 5.0
    T = np.zeros((3, 4), np.float32); T[0, 0] = T[1, 1] = T[2, 2] = 1; T[0, 3] = 5 * 5.0 / 1000.0; T[1, 3] = -3 * 5.0 / 1000.0
    lat = []
    for _ in range(12):
        t0 = time.perf_counter()
        nm, _ = M.search_by_projection_frames(m, [v1], [v0], [np.ones(len(k0), np.uint8)], [np.zeros(len(k0), np.uint8)], [world], [T],
                                              1000.0, 1000.0, 960.0, 540.0, 15.0)
        lat.append((time.perf_counter() - t0) * 1e3)
    prev = np.stack([k0["x"], k0["y"]], axis=1).astype(np.float32)
    n8, _, _ = M.search_for_initialization(m, v0, v1, prev, 100)
    n7, _ = M.window_search(m, v0, v1, np.ones(len(k0), np.uint8), 50)
    out = {"sbp_single_pair_host_call_ms_median": float(np.median(lat[2:])), "sbp_matches": int(nm[0]), "init_matches": int(n8),
           "window_matches": int(n7)}
    try:
        V = BW.Vocabulary(random_vocabulary(10, 4, seed=3))
        out["bow_words"] = int(len(V.transform(d0, 2)[0][0]))
        gp = np.arange(0, len(d0) + 1, 20, dtype=np.int32)
        out["distinctive_groups"] = int(len(BW.distinctive_descriptors(m, d0[:gp[-1]], gp)))
        # feature_vector_kernel and search_by_bow_kernel: frame 1 against frame 0, device-resident
        dev = torch.device("cuda", 0)
        cap = 2000
        kk, dd = np.zeros((2, cap), fe.KP_DTYPE), np.zeros((2, cap, 32), np.uint8)
        kk[0, :len(k0)], kk[1, :len(k1)], dd[0, :len(d0)], dd[1, :len(d1)] = k0, k1, d0, d1
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        d_k, d_d, d_c = t(kk.view(np.uint8).reshape(2, cap, 28)), t(dd), t(np.array([len(k0), len(k1)], np.int32))
        d_leaf, d_node = (torch.zeros(2 * cap, dtype=torch.int32, device=dev) for _ in range(2))
        d_ids, d_items, d_out = (torch.zeros((2, cap), dtype=torch.int32, device=dev) for _ in range(3))
        d_ptr, d_n = torch.zeros((2, cap + 1), dtype=torch.int32, device=dev), torch.zeros(2, dtype=torch.int32, device=dev)
        d_valid, d_i1, d_i2 = torch.ones((2, cap), dtype=torch.uint8, device=dev), t(np.array([1], np.int32)), t(np.array([0], np.int32))
        d_nm = torch.zeros(1, dtype=torch.int32, device=dev)
        s = torch.cuda.Stream(device=dev)
        torch.cuda.synchronize()
        V.descend_device(d_d.data_ptr(), 2 * cap, 2, d_leaf.data_ptr(), d_node.data_ptr(), s.cuda_stream)
        BW.feature_vector_device(V, 2, d_leaf.data_ptr(), d_node.data_ptr(), d_c.data_ptr(), cap, d_ids.data_ptr(), d_ptr.data_ptr(),
                                 d_items.data_ptr(), d_n.data_ptr(), s.cuda_stream)
        M.search_by_bow_device(m, 0, 1, d_k.data_ptr(), d_d.data_ptr(), d_c.data_ptr(), cap, d_ids.data_ptr(), d_ptr.data_ptr(),
                               d_items.data_ptr(), d_n.data_ptr(), d_valid.data_ptr(), d_i1.data_ptr(), d_i2.data_ptr(), d_out.data_ptr(),
                               d_nm.data_ptr(), s.cuda_stream)
        s.synchronize()
        m.sync()
        out["bow_device_matches"] = int(d_nm.item())
        # search_for_triangulation_kernel: frame 0 against frame 1 (shifted by (5, -3): epipolar line y2 = y1 - 3)
        d_F = t(np.array([[0, 0, 0, 0, 0, -1, 0, 1, 3]], np.float32))
        d_mp = torch.zeros((2, cap), dtype=torch.uint8, device=dev)
        sigma2 = (np.float32(1.2) ** np.arange(8, dtype=np.float32)) ** 2
        M.search_for_triangulation_device(m, 1, d_k.data_ptr(), d_d.data_ptr(), d_c.data_ptr(), cap, d_ids.data_ptr(), d_ptr.data_ptr(),
                                          d_items.data_ptr(), d_n.data_ptr(), d_mp.data_ptr(), d_i2.data_ptr(), d_i1.data_ptr(),
                                          d_F.data_ptr(), sigma2, d_out.data_ptr(), d_nm.data_ptr(), s.cuda_stream)
        s.synchronize()
        m.sync()
        out["triangulation_device_matches"] = int(d_nm.item())
        # distinctive_kernel<true>: the same groups as above, addressed through observation slots of frame 0
        d_gp, d_obs = t(gp), t(np.arange(gp[-1], dtype=np.int32))
        d_best, d_mpd = torch.zeros(len(gp) - 1, dtype=torch.int32, device=dev), torch.zeros((len(gp) - 1, 32), dtype=torch.uint8, device=dev)
        BW.distinctive_descriptors_device(m, len(gp) - 1, d_d.data_ptr(), d_c.data_ptr(), 2, cap, d_gp.data_ptr(), d_obs.data_ptr(),
                                          int(gp[-1]), d_best.data_ptr(), d_mpd.data_ptr(), s.cuda_stream)
        s.synchronize()
        m.sync()
        out["distinctive_device_groups"] = int((d_best >= 0).sum().item())
        V.close()
    except Exception as e:
        out["bow"] = "skipped: %r" % e
    ex.close(); m.close()
    return out


def reloc(args):
    import torch
    import orb_slam_b200 as fe
    from orb_slam_b200 import matching as M, bow as BW
    from orb_slam_b200.synth import textured_frame, shifted_frame, random_vocabulary
    W, H, NF, levelsup, NKF, NLOOP = 1920, 1080, 2000, 4, 32, 16
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    s = stream.cuda_stream
    base = textured_frame(W, H, seed=21)
    # frame 0: the current frame; frames 1..32: the candidate keyframes (views of the same place)
    frames = np.stack([base] + [shifted_frame(base, 4 * (i % 5) - 8, 3 * (i % 3) - 3, seed=i) for i in range(1, NKF + 1)])
    F = len(frames)
    ex = fe.ORBextractor(NF, 1.2, 8)
    kps, desc, cnt = ex.extract_batch(frames)
    ex.close()
    voc = random_vocabulary(10, 6, seed=3)   # the shape of ORBvoc: k = 10, L = 6; levelsup 4 = nodes of level 2
    V = BW.Vocabulary(voc)
    valid = (np.random.default_rng(1).random((F, NF)) < 0.9).astype(np.uint8)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d_k, d_d, d_c, d_valid = t(kps.view(np.uint8).reshape(F, NF, 28)), t(desc), t(cnt), t(valid)
    d_leaf, d_node = (torch.zeros(F * NF, dtype=torch.int32, device=dev) for _ in range(2))
    d_ids, d_items = (torch.zeros((F, NF), dtype=torch.int32, device=dev) for _ in range(2))
    d_ptr, d_n = torch.zeros((F, NF + 1), dtype=torch.int32, device=dev), torch.zeros(F, dtype=torch.int32, device=dev)
    m = fe.ORBmatcher(0.75, True)
    V.descend_device(d_d.data_ptr(), F * NF, levelsup, d_leaf.data_ptr(), d_node.data_ptr(), s)

    def timed(fn, iters=args.iters * 4, warm=args.warmup):
        for _ in range(warm):
            fn()
        stream.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(iters):
            fn()
        e1.record(stream)
        stream.synchronize()
        return e0.elapsed_time(e1) / iters

    out = {"what": "SearchByBoW device-resident, 1920x1080 frames, %d keypoints, vocabulary k=10 L=6, levelsup %d" % (NF, levelsup),
           "counts_min": int(cnt.min())}
    fv = lambda nf: BW.feature_vector_device(V, nf, d_leaf.data_ptr(), d_node.data_ptr(), d_c.data_ptr(), NF, d_ids.data_ptr(),
                                             d_ptr.data_ptr(), d_items.data_ptr(), d_n.data_ptr(), s)
    out["feature_vector_1_frame_ms"] = timed(lambda: fv(1))
    out["feature_vector_%d_frames_ms" % F] = timed(lambda: fv(F))
    stream.synchronize()
    ids, ptr, items, nn = (x.cpu().numpy() for x in (d_ids, d_ptr, d_items, d_n))
    fvs = [(ids[f, :nn[f]], ptr[f, :nn[f] + 1], items[f, :ptr[f, nn[f]]]) for f in range(F)]
    out["nodes_per_frame_mean"] = float(nn.mean())
    for tag, variant, jobs in (("reloc_%dkf" % NKF, 0, [(f, 0) for f in range(1, NKF + 1)]),
                               ("loop_%dcand" % NLOOP, 1, [(0, f) for f in range(1, NLOOP + 1)])):
        j = np.array(jobs, np.int32)
        d_i1, d_i2 = t(j[:, 0]), t(j[:, 1])
        d_out = torch.zeros((len(j), NF), dtype=torch.int32, device=dev)
        d_nm = torch.zeros(len(j), dtype=torch.int32, device=dev)
        call = lambda: M.search_by_bow_device(m, variant, len(j), d_k.data_ptr(), d_d.data_ptr(), d_c.data_ptr(), NF, d_ids.data_ptr(),
                                              d_ptr.data_ptr(), d_items.data_ptr(), d_n.data_ptr(), d_valid.data_ptr(), d_i1.data_ptr(),
                                              d_i2.data_ptr(), d_out.data_ptr(), d_nm.data_ptr(), s)
        out[tag + "_device_ms"] = timed(call)
        m.sync()
        dev_out, dev_nm = d_out.cpu().numpy(), d_nm.cpu().numpy()
        same = True
        lat = []
        for rep in range(3):
            t0 = time.perf_counter()
            for q, (f1, f2) in enumerate(jobs):
                n1, n2 = cnt[f1], cnt[f2]
                nm, o = M.search_by_bow(m, variant, desc[f1, :n1], valid[f1, :n1], kps[f1, :n1]["angle"], fvs[f1], desc[f2, :n2],
                                        valid[f2, :n2], kps[f2, :n2]["angle"], fvs[f2])
                if rep == 0:
                    same = same and nm == dev_nm[q] and np.array_equal(o, dev_out[q, :len(o)])
            lat.append((time.perf_counter() - t0) * 1e3)
        out[tag + "_host_per_pair_wall_ms"] = float(np.median(lat))
        out[tag + "_matches"] = int(dev_nm.sum())
        out[tag + "_same_as_host"] = bool(same)
    V.close(); m.close()
    return out


def mapping(args):
    """SearchForTriangulation at its call site, LocalMapping::CreateNewMapPoints (LocalMapping.cc:205-252): the new keyframe
    against its 20 covisible neighbours, ORBmatcher(0.6, false).  The neighbours are sideways camera moves (R = I, t = (tx, 0,
    0)) seen as horizontal image shifts, and F12 is computed from the poses as ComputeF12 does (LocalMapping.cc:452-469)."""
    import torch
    import orb_slam_b200 as fe
    from orb_slam_b200 import matching as M, bow as BW
    from orb_slam_b200.synth import textured_frame, shifted_frame, random_vocabulary
    W, H, NF, levelsup, NKF = 1920, 1080, 2000, 4, 20
    fx = fy = 1000.0
    cx, cy = 960.0, 540.0
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    s = stream.cuda_stream
    base = textured_frame(W, H, seed=23)
    dxs = [0] + [(-1) ** i * (2 + i % 7) for i in range(1, NKF + 1)]   # never 0: every neighbour passes the baseline test
    frames = np.stack([base] + [shifted_frame(base, dxs[i], 0, seed=i) for i in range(1, NKF + 1)])
    F = len(frames)
    ex = fe.ORBextractor(NF, 1.2, 8)
    kps, desc, cnt = ex.extract_batch(frames)
    ex.close()
    voc = random_vocabulary(10, 6, seed=3)
    V = BW.Vocabulary(voc)
    has_mp = (np.random.default_rng(2).random((F, NF)) < 0.3).astype(np.uint8)
    sigma2 = (np.float32(1.2) ** np.arange(8, dtype=np.float32)) ** 2
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)
    Kinv = np.linalg.inv(K).astype(np.float32)
    F12 = np.zeros((NKF, 9), np.float32)
    for j in range(NKF):   # pKF1 = frame 0 at the origin, pKF2 = frame j + 1 with R2w = I, t2w = (dx / fx * depth, 0, 0), depth 5
        t12 = -np.array([dxs[j + 1] / fx * 5.0, 0, 0], np.float32)   # -R1w R2w^T t2w + t1w
        t12x = np.array([[0, -t12[2], t12[1]], [t12[2], 0, -t12[0]], [-t12[1], t12[0], 0]], np.float32)
        F12[j] = (Kinv.T @ t12x @ np.eye(3, dtype=np.float32) @ Kinv).reshape(-1)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d_k, d_d, d_c, d_mp, d_F = t(kps.view(np.uint8).reshape(F, NF, 28)), t(desc), t(cnt), t(has_mp), t(F12)
    d_leaf, d_node = (torch.zeros(F * NF, dtype=torch.int32, device=dev) for _ in range(2))
    d_ids, d_items = (torch.zeros((F, NF), dtype=torch.int32, device=dev) for _ in range(2))
    d_ptr, d_n = torch.zeros((F, NF + 1), dtype=torch.int32, device=dev), torch.zeros(F, dtype=torch.int32, device=dev)
    V.descend_device(d_d.data_ptr(), F * NF, levelsup, d_leaf.data_ptr(), d_node.data_ptr(), s)
    BW.feature_vector_device(V, F, d_leaf.data_ptr(), d_node.data_ptr(), d_c.data_ptr(), NF, d_ids.data_ptr(), d_ptr.data_ptr(),
                             d_items.data_ptr(), d_n.data_ptr(), s)
    stream.synchronize()
    ids, ptr, items, nn = (x.cpu().numpy() for x in (d_ids, d_ptr, d_items, d_n))
    fvs = [(ids[f, :nn[f]], ptr[f, :nn[f] + 1], items[f, :ptr[f, nn[f]]]) for f in range(F)]
    jobs = [(0, f) for f in range(1, NKF + 1)]
    j = np.array(jobs, np.int32)
    d_i1, d_i2 = t(j[:, 0]), t(j[:, 1])
    d_out = torch.zeros((NKF, NF), dtype=torch.int32, device=dev)
    d_nm = torch.zeros(NKF, dtype=torch.int32, device=dev)
    m = fe.ORBmatcher(0.6, False)   # LocalMapping.cc:210
    call = lambda: M.search_for_triangulation_device(m, NKF, d_k.data_ptr(), d_d.data_ptr(), d_c.data_ptr(), NF, d_ids.data_ptr(),
                                                     d_ptr.data_ptr(), d_items.data_ptr(), d_n.data_ptr(), d_mp.data_ptr(),
                                                     d_i1.data_ptr(), d_i2.data_ptr(), d_F.data_ptr(), sigma2, d_out.data_ptr(),
                                                     d_nm.data_ptr(), s)
    for _ in range(args.warmup):
        call()
    stream.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    iters = args.iters * 4
    e0.record(stream)
    for _ in range(iters):
        call()
    e1.record(stream)
    stream.synchronize()
    m.sync()
    out = {"what": "SearchForTriangulation device-resident, 1920x1080 keyframe, %d keypoints, against %d neighbours, vocabulary "
                   "k=10 L=6, levelsup %d" % (NF, NKF, levelsup),
           "counts_min": int(cnt.min()), "nodes_per_frame_mean": float(nn.mean()),
           "mapping_%dkf_device_ms" % NKF: e0.elapsed_time(e1) / iters}
    dev_out, dev_nm = d_out.cpu().numpy(), d_nm.cpu().numpy()
    same = True
    lat = []
    for rep in range(3):
        t0 = time.perf_counter()
        for q, (f1, f2) in enumerate(jobs):
            n1, n2 = cnt[f1], cnt[f2]
            nm, o = M.search_for_triangulation(m, kps[f1, :n1], desc[f1, :n1], has_mp[f1, :n1], fvs[f1], kps[f2, :n2], desc[f2, :n2],
                                               has_mp[f2, :n2], fvs[f2], F12[q], sigma2)
            if rep == 0:
                same = same and nm == dev_nm[q] and np.array_equal(o, dev_out[q, :len(o)])
        lat.append((time.perf_counter() - t0) * 1e3)
    out["mapping_%dkf_host_per_pair_wall_ms" % NKF] = float(np.median(lat))
    out["mapping_%dkf_matches" % NKF] = int(dev_nm.sum())
    out["same_as_host"] = bool(same)
    _gpu_and_power_limit(out)
    V.close(); m.close()
    return out


def _gpu_and_power_limit(out):
    try:
        import subprocess
        import torch
        out["gpu"] = torch.cuda.get_device_properties(0).name
        out["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                                            capture_output=True, text=True).stdout.strip()
    except Exception as e:
        out["gpu"] = "unknown: %r" % e


def mapdesc(args):
    """MapPoint::ComputeDistinctiveDescriptors at LocalMapping::ProcessNewKeyFrame (LocalMapping.cc:150): every feature of one
    keyframe of 2000 features (the 1080p configuration's keypoint count) is a map point, observed in a store of 60 keyframes
    of 2000 features.  Observation counts come from a fixed seeded distribution (95 % in 2-10, 5 % in 11-150); the "tail"
    run adds one map point with 1000 observations.  The descriptors are synthetic: the observations of one point are noisy
    copies of one random descriptor, every other row is random.  CUDA-event ms of
    orbfe_distinctive_descriptors_device, next to the wall time of the same groups through orbfe_distinctive_descriptors
    including the host gather of their descriptors from a host copy of the store, and same_as_host."""
    import torch
    import orb_slam_b200 as fe
    from orb_slam_b200 import bow as BW
    from orb_slam_b200.synth import noisy_copies, random_descriptors
    NKF, NF = 60, 2000
    rng = np.random.default_rng(13)
    store = random_descriptors(NKF * NF, 13).reshape(NKF, NF, 32)
    counts = np.full(NKF, NF, np.int32)
    free = [list(rng.permutation(NF)) for _ in range(NKF)]   # frame 0: the new keyframe, its feature p is map point p
    free[0] = []
    n_obs = np.where(rng.random(NF) < 0.95, rng.integers(2, 11, NF), rng.integers(11, 151, NF))
    groups = []
    for p in range(NF + 1):
        tail = p == NF
        k = 1000 if tail else int(n_obs[p]) - 1   # observations outside the new keyframe
        frames = np.sort(rng.choice(np.arange(1, NKF), k, replace=k > NKF - 1))
        g = ([] if tail else [p]) + [int(f) * NF + int(free[f].pop()) for f in frames]   # mObservations order: by keyframe
        base = random_descriptors(1, 50000 + p)
        store.reshape(-1, 32)[g] = noisy_copies(np.repeat(base, len(g), axis=0), 0.12, 60000 + p)
        groups.append(np.array(g, np.int32))
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    s = stream.cuda_stream
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d_desc, d_cnt = t(store), t(counts)
    m = fe.ORBmatcher(0.6, True)
    out = {"what": "ComputeDistinctiveDescriptors device-resident: the %d map points of one keyframe over a %d-keyframe store of %d "
                   "features" % (NF, NKF, NF)}
    for tag, gs in (("kf", groups[:NF]), ("kf_tail1000", groups)):
        ptr = np.concatenate([[0], np.cumsum([len(g) for g in gs])]).astype(np.int32)
        obs = np.concatenate(gs).astype(np.int32)
        ng = len(gs)
        d_ptr, d_obs = t(ptr), t(obs)
        d_best, d_mp = torch.zeros(ng, dtype=torch.int32, device=dev), torch.zeros((ng, 32), dtype=torch.uint8, device=dev)
        call = lambda: BW.distinctive_descriptors_device(m, ng, d_desc.data_ptr(), d_cnt.data_ptr(), NKF, NF, d_ptr.data_ptr(),
                                                         d_obs.data_ptr(), len(obs), d_best.data_ptr(), d_mp.data_ptr(), s)
        for _ in range(args.warmup):
            call()
        stream.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        iters = args.iters * 4
        e0.record(stream)
        for _ in range(iters):
            call()
        e1.record(stream)
        stream.synchronize()
        m.sync()
        out[tag + "_device_ms"] = e0.elapsed_time(e1) / iters
        out[tag + "_groups"], out[tag + "_observations"], out[tag + "_max_group"] = ng, int(len(obs)), int(np.diff(ptr).max())
        lat, best_h = [], None
        flat = store.reshape(-1, 32)
        for _ in range(5):
            t0 = time.perf_counter()
            best_h = BW.distinctive_descriptors(m, flat[obs], ptr)
            lat.append((time.perf_counter() - t0) * 1e3)
        out[tag + "_host_entry_with_gather_wall_ms"] = float(np.median(lat))
        best = d_best.cpu().numpy()
        out[tag + "_same_as_host"] = bool(np.array_equal(best, best_h) and np.array_equal(d_mp.cpu().numpy(), flat[obs[ptr[:-1] + best]]))
    _gpu_and_power_limit(out)
    m.close()
    return out


def matchers(args):
    """Device-resident matcher calls timed with CUDA events: SearchByProjection(Frame,Frame) for 1 and 64 pairs at 1080p / 2000 kp,
    SearchForInitialization for 8 pairs at 720p (config 4's matcher)."""
    import torch
    import orb_slam_b200 as fe
    from orb_slam_b200 import matching as M
    from orb_slam_b200.synth import textured_frame, shifted_frame
    dev = torch.device("cuda", 0)
    out = {}
    stream = torch.cuda.Stream(device=dev)
    s = stream.cuda_stream

    def timed(fn, iters=20, warm=5):
        for _ in range(warm):
            fn()
        stream.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(iters):
            fn()
        e1.record(stream)
        stream.synchronize()
        return e0.elapsed_time(e1) / iters
    # ---- M2 at the bench geometry
    W, H, NF = 1920, 1080, 2000
    f0 = textured_frame(W, H, seed=9)
    frames = np.stack([f0] + [shifted_frame(f0, 3 * (i % 3) - 3, 2 * (i % 2) - 1, seed=i) for i in range(1, 9)])
    ex = fe.ORBextractor(NF, 1.2, 8)
    kps, desc, cnt = ex.extract_batch(frames)
    ex.close()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    world = np.zeros((9, NF, 3), np.float32)
    world[:, :, 0] = (kps["x"] - 960.0) / 1000.0 * 5.0; world[:, :, 1] = (kps["y"] - 540.0) / 1000.0 * 5.0; world[:, :, 2] = 5.0
    d_kps, d_desc, d_cnt = t(kps.view(np.uint8).reshape(9, NF, 28)), t(desc), t(cnt)
    d_world, d_flags = t(world), torch.ones((9, NF), dtype=torch.uint8, device=dev)
    m = fe.ORBmatcher(0.9, True)
    for npairs in (1, 8, 64):
        cur = np.array([1 + (j % 8) for j in range(npairs)], np.int32)
        last = cur - 1
        T = np.tile(np.array([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0], np.float32), (npairs, 1))
        d_cur, d_last, d_T = t(cur), t(last), t(T)
        d_mp = torch.full((npairs, NF), -1, dtype=torch.int32, device=dev)
        d_nm = torch.zeros(npairs, dtype=torch.int32, device=dev)

        def call():
            d_mp.fill_(-1)
            M.search_by_projection_device(m, npairs, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), NF, d_cur.data_ptr(), d_last.data_ptr(),
                                          d_world.data_ptr(), d_flags.data_ptr(), d_T.data_ptr(), W, H, 1.2, 8, 1000.0, 1000.0, 960.0, 540.0, 15.0,
                                          d_mp.data_ptr(), d_nm.data_ptr(), s)
        with torch.cuda.stream(stream):
            out["sbp_ff_%d_pairs_ms" % npairs] = timed(call)
        out["sbp_ff_%d_pairs_matches" % npairs] = int(d_nm.sum().item())
    # ---- M8 at the rig geometry
    W2, H2 = 1280, 720
    g0 = textured_frame(W2, H2, seed=40)
    fr2 = np.stack([g0, shifted_frame(g0, 12, 4, seed=1)])
    ex2 = fe.ORBextractor(NF, 1.2, 8)
    k2, dd2, c2 = ex2.extract_batch(fr2)
    ex2.close()
    d_k2, d_d2, d_c2 = t(k2.view(np.uint8).reshape(2, NF, 28)), t(dd2), t(c2)
    for npairs in (1, 8):
        f1 = t(np.zeros(npairs, np.int32)); f2 = t(np.ones(npairs, np.int32))
        prev0 = np.tile(np.stack([k2[0]["x"], k2[0]["y"]], axis=1).astype(np.float32)[None], (npairs, 1, 1))
        d_prev0, d_prev = t(prev0), t(prev0)
        d_m12 = torch.full((npairs, NF), -1, dtype=torch.int32, device=dev); d_nm2 = torch.zeros(npairs, dtype=torch.int32, device=dev)

        def call2():
            d_prev.copy_(d_prev0)
            M.search_for_initialization_device(m, npairs, d_k2.data_ptr(), d_d2.data_ptr(), d_c2.data_ptr(), NF, f1.data_ptr(), f2.data_ptr(),
                                               d_prev.data_ptr(), W2, H2, 100, d_m12.data_ptr(), d_nm2.data_ptr(), s)
        with torch.cuda.stream(stream):
            out["init_%d_pairs_ms" % npairs] = timed(call2)
        out["init_%d_pairs_matches" % npairs] = int(d_nm2.sum().item())
    m.close()
    return out


def windowed(args):
    """The host-array windowed matchers one call at a time, as ORB-SLAM's tracking thread calls them: median wall ms per call
    over `--iters` x 10 calls after `--warmup` calls."""
    import orb_slam_b200 as fe
    from orb_slam_b200 import matching as M
    from orb_slam_b200.synth import textured_frame, shifted_frame
    NF = 2000
    out = {}

    def wall(fn):
        for _ in range(args.warmup):
            fn()
        lat = []
        for _ in range(args.iters * 10):
            t0 = time.perf_counter()
            fn()
            lat.append((time.perf_counter() - t0) * 1e3)
        return float(np.median(lat))
    W, H, fx, cx, cy, depth = 1920, 1080, 1000.0, 960.0, 540.0, 5.0
    f0 = textured_frame(W, H, seed=9)
    frames = np.stack([f0] + [shifted_frame(f0, 3 * (i % 3) - 3, 2 * (i % 2) - 1, seed=i) for i in range(1, 9)])
    ex = fe.ORBextractor(NF, 1.2, 8)
    kps, desc, cnt = ex.extract_batch(frames)
    ex.close()
    views = [M.FrameView(kps[f, :cnt[f]], desc[f, :cnt[f]], W, H) for f in range(9)]
    world = [np.stack([(kps[f]["x"] - cx) / fx * depth, (kps[f]["y"] - cy) / fx * depth, np.full(NF, depth)], 1).astype(np.float32)
             for f in range(9)]
    ones, zeros, T = np.ones(NF, np.uint8), np.zeros(NF, np.uint8), np.eye(3, 4, dtype=np.float32)
    m = fe.ORBmatcher(0.9, True)
    for npairs in (1, 8):
        call = lambda: M.search_by_projection_frames(m, views[1:npairs + 1], views[:npairs], [ones] * npairs, [zeros] * npairs,
                                                     world[:npairs], [T] * npairs, fx, fx, cx, cy, 15.0)
        out["sbp_frames_%d_pairs_wall_ms" % npairs] = wall(call)
        out["sbp_frames_%d_pairs_matches" % npairs] = int(call()[0].sum())
    k0, k1 = kps[0, :cnt[0]], kps[1, :cnt[1]]
    proj = np.stack([k0["x"], k0["y"]], 1).astype(np.float32)
    call = lambda: M.search_local_points(m, views[1], ones[:len(k0)], proj, k0["octave"], np.full(len(k0), 0.999, np.float32),
                                         desc[0, :cnt[0]], 1.0)
    out["local_points_wall_ms"], out["local_points_matches"] = wall(call), call()[0]
    call = lambda: M.window_search(m, views[0], views[1], ones[:len(k0)], 50)
    out["window_search_wall_ms"], out["window_search_matches"] = wall(call), call()[0]
    W2, H2 = 1280, 720
    g0 = textured_frame(W2, H2, seed=40)
    ex2 = fe.ORBextractor(NF, 1.2, 8)
    k2, d2, c2 = ex2.extract_batch(np.stack([g0, shifted_frame(g0, 12, 4, seed=1)]))
    ex2.close()
    v1, v2 = M.FrameView(k2[0, :c2[0]], d2[0, :c2[0]], W2, H2), M.FrameView(k2[1, :c2[1]], d2[1, :c2[1]], W2, H2)
    prev = np.stack([k2[0]["x"][:c2[0]], k2[0]["y"][:c2[0]]], 1).astype(np.float32)
    call = lambda: M.search_for_initialization(m, v1, v2, prev, 100)
    out["init_720p_wall_ms"], out["init_720p_matches"] = wall(call), call()[0]
    m.close()
    _gpu_and_power_limit(out)
    return out


def exchange1(args):
    """The exchange variant of the descriptor kernel with a world of ONE rank (its peer table holds only this GPU): what the
    remote-store code path, the acknowledgement poll and the publish cost by themselves, without NVLink or a second rank."""
    import torch
    import torch.distributed as dist
    import orb_slam_b200 as fe
    from orb_slam_b200 import comm as CM
    from orb_slam_b200.synth import textured_frame
    W, H, NF, T = 1280, 720, 2000, 8
    dev = torch.device("cuda", 0)
    frames = np.stack([textured_frame(W, H, seed=40 + t) for t in range(T)])
    d_frames = torch.from_numpy(frames).to(dev)
    ex = fe.ORBextractor(NF, 1.2, 8)
    comm = CM.Comm.create(torch, dist, 0)
    x = CM.RigExchange(comm, NF, T)
    d_kps = torch.zeros((T, NF, 28), dtype=torch.uint8, device=dev)
    d_desc = torch.zeros((T, NF, 32), dtype=torch.uint8, device=dev)
    d_cnt = torch.zeros((T,), dtype=torch.int32, device=dev)
    stream = torch.cuda.Stream(device=dev)
    s = stream.cuda_stream

    def plain():
        ex.extract_batch_device(d_frames.data_ptr(), W, H, W, W * H, T, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), s)

    def exch():
        x.extract(ex, d_frames.data_ptr(), W, H, W, W * H, s)

    out = {"what": "exchange variant of describe_fused with world = 1 (8 x 1280x720, 2000 kp)"}
    ex.set_profiling(True)
    for name, fn in (("plain", plain), ("exchange_self", exch), ("plain_again", plain)):
        for _ in range(args.warmup):
            fn()
        stream.synchronize()
        ex.stage_times()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.iters):
            fn()
        e1.record(stream)
        stream.synchronize()
        acc = {}
        for k, v in ex.stage_times():
            acc[k] = acc.get(k, 0.0) + v / args.iters
        out[name] = {"ms_per_call": e0.elapsed_time(e1) / args.iters, "describe_ms": acc.get("describe")}
    x.close(); comm.close(); ex.close()
    return out


def h2d(args):
    """Raw pinned-host -> device copy bandwidth of this box (64 frames of 1080p per copy burst), with the pinned buffer
    allocated from wherever the process runs and again after moving the process to the GPU's NUMA node: what the e2e
    number of bench.py can reach at best on this host."""
    import os
    import torch
    dev = torch.device("cuda", 0)
    out = {}
    n = 64 * 1920 * 1080
    dst = torch.empty(n, dtype=torch.uint8, device=dev)

    def probe(tag):
        src = torch.empty(n, dtype=torch.uint8).pin_memory()
        src.fill_(3)
        res = torch.empty(4 << 20, dtype=torch.uint8).pin_memory()
        for _ in range(3):
            dst.copy_(src, non_blocking=True)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            dst.copy_(src, non_blocking=True)
        e1.record(); torch.cuda.synchronize()
        out["h2d_GBps_" + tag] = 10 * n / (e0.elapsed_time(e1) * 1e-3) / 1e9
        e0.record()
        for _ in range(10):
            for f in range(64):
                dst[f * 1920 * 1080:(f + 1) * 1920 * 1080].copy_(src[f * 1920 * 1080:(f + 1) * 1920 * 1080], non_blocking=True)
        e1.record(); torch.cuda.synchronize()
        out["h2d_GBps_per_frame_copies_" + tag] = 10 * n / (e0.elapsed_time(e1) * 1e-3) / 1e9
        e0.record()
        for _ in range(10):
            res.copy_(dst[:4 << 20], non_blocking=True)
        e1.record(); torch.cuda.synchronize()
        out["d2h_GBps_4MB_" + tag] = 10 * (4 << 20) / (e0.elapsed_time(e1) * 1e-3) / 1e9
    probe("as_started")
    try:
        pr = torch.cuda.get_device_properties(0)
        bdf = "%04x:%02x:%02x.0" % (getattr(pr, "pci_domain_id", 0), pr.pci_bus_id, pr.pci_device_id)
        out["gpu_numa_node"] = open("/sys/bus/pci/devices/%s/numa_node" % bdf).read().strip()
        txt = open("/sys/bus/pci/devices/%s/local_cpulist" % bdf).read().strip()
        out["gpu_local_cpulist"] = txt
        out["started_on_cpu"] = os.sched_getcpu() if hasattr(os, "sched_getcpu") else None
        cpus = set()
        for part in txt.split(","):
            a, _, b = part.partition("-")
            cpus |= set(range(int(a), int(b or a) + 1))
        os.sched_setaffinity(0, cpus & set(os.sched_getaffinity(0)))
        probe("on_gpu_node")
    except Exception as e:
        out["numa_probe_error"] = repr(e)
    return out


def fast(args):
    """BASELINE configs[1] geometry (1920x1080, 2000 kp, 8 levels), 64-frame device-resident batches: per-stage CUDA-event
    times of the extractor, the FAST kernel's stage included."""
    import torch
    import orb_slam_b200 as fe
    from orb_slam_b200.synth import textured_frame, shifted_frame
    W, H, NF, NL, B = 1920, 1080, 2000, 8, 64
    bases = [textured_frame(W, H, seed=100 + i) for i in range(4)]
    frames = np.stack([shifted_frame(bases[i % 4], 2 * i, i, seed=i) for i in range(B)])
    dev = torch.device("cuda", 0)
    d_frames = torch.from_numpy(frames).to(dev)
    d_kps = torch.empty((B, NF, 28), dtype=torch.uint8, device=dev)
    d_desc = torch.empty((B, NF, 32), dtype=torch.uint8, device=dev)
    d_cnt = torch.empty((B,), dtype=torch.int32, device=dev)
    stream = torch.cuda.Stream(device=dev)
    out = {"what": "FAST kernel, 1080p x 64 frames, ms per batch"}
    ex = fe.ORBextractor(NF, 1.2, NL, fe.FAST_SCORE, 20)
    ex.set_profiling(True)
    for _ in range(3):
        ex.extract_batch_device(d_frames.data_ptr(), W, H, W, W * H, B, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), stream.cuda_stream)
    stream.synchronize()
    ex.stage_times()
    n = 10
    for rep in range(2):
        for _ in range(n):
            ex.extract_batch_device(d_frames.data_ptr(), W, H, W, W * H, B, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), stream.cuda_stream)
        stream.synchronize()
        acc = {}
        for name, ms in ex.stage_times():
            acc[name] = acc.get(name, 0.0) + ms / n
        out["rep%d" % rep] = {"fast_nms": round(acc.get("fast_nms", -1), 4), "all": round(sum(acc.values()), 4),
                              "stages": {k: round(v, 4) for k, v in acc.items()}}
    ex.close()
    return out


def latency(args):
    """Small-batch shapes, per-stage CUDA-event times of the device-resident extractor: one 1080p frame (the reference's own call
    shape) and eight 720p frames (one rig step of configs[3])."""
    import torch
    import orb_slam_b200 as fe
    from orb_slam_b200.synth import textured_frame, shifted_frame
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    out = {"what": "per-stage ms of small extractor batches (device-resident)"}
    for tag, W, H, B in (("1x1080p", 1920, 1080, 1), ("8x720p", 1280, 720, 8)):
        base = textured_frame(W, H, seed=5)
        frames = np.stack([shifted_frame(base, 2 * i, i, seed=i) for i in range(B)])
        d_frames = torch.from_numpy(frames).to(dev)
        d_kps = torch.empty((B, 2000, 28), dtype=torch.uint8, device=dev)
        d_desc = torch.empty((B, 2000, 32), dtype=torch.uint8, device=dev)
        d_cnt = torch.empty((B,), dtype=torch.int32, device=dev)
        ex = fe.ORBextractor(2000, 1.2, 8, fe.FAST_SCORE, 20)
        call = lambda: ex.extract_batch_device(d_frames.data_ptr(), W, H, W, W * H, B, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(),
                                               stream.cuda_stream)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n = 50
        for _ in range(5):
            call()
        stream.synchronize()
        with torch.cuda.stream(stream):      # no stage events between the kernels: what a caller sees
            e0.record(stream)
            for _ in range(n):
                call()
            e1.record(stream)
        stream.synchronize()
        ms_plain = e0.elapsed_time(e1) / n
        ex.set_profiling(True)
        for _ in range(3):
            call()
        stream.synchronize()
        ex.stage_times()
        for _ in range(n):
            call()
        stream.synchronize()
        acc = {}
        for name, ms in ex.stage_times():
            acc[name] = acc.get(name, 0.0) + ms / n
        out[tag] = {"ms_per_call": ms_plain, "pdl": os.environ.get("ORBFE_PDL", "1"), "stages": {k: round(v, 4) for k, v in acc.items()}}
        ex.close()
    return out


def kfdb(args):
    """The resident keyframe database (orbfe_kfdb_*) at 1k and 10k keyframes of about 1000 words each, word ids spread over
    10^6 (the size of ORBvoc): device time per loop and per relocalisation query (CUDA events around orbfe_kfdb_detect_device,
    queries taken from the keyframes' own neighbourhood so that candidates exist), host time per add and per erase (both
    synchronous), and on the same data the wall time of the stateless orbfe_bow_db_detect (CSR arrays of the whole
    database uploaded per query)."""
    import time
    import torch
    import orb_slam_b200 as fe
    from orb_slam_b200 import bow as BW
    NW, WPK = 1_000_000, 1000
    n = NW + 1
    cp = np.zeros(n + 1, np.int32)
    cp[1:] = NW
    V = BW.Vocabulary({"node_desc": np.zeros((n, 32), np.uint8), "child_ptr": cp, "children": np.arange(1, n, dtype=np.int32),
                       "word_id": np.arange(-1, NW, dtype=np.int32), "weight": np.ones(n), "L": 1})
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    m = fe.ORBmatcher(0.75, True)
    out = {"what": "KeyFrameDatabase resident on the device: %d words per keyframe, word ids over 10^6" % WPK}
    _gpu_and_power_limit(out)
    for nkf in (1000, 10000):
        rng = np.random.default_rng(nkf)
        shift = 100
        track = rng.integers(0, NW, nkf * shift + 4 * WPK)

        def bow_at(pos):
            w = track[pos:pos + WPK].copy()
            flip = rng.random(WPK) < 0.25
            w[flip] = rng.integers(0, NW, int(flip.sum()))
            ids = np.unique(w).astype(np.int32)
            v = rng.uniform(0.2, 3.0, len(ids))
            return ids, v / v.sum()

        bows = [bow_at(shift * k) for k in range(nkf)]
        db = BW.KeyFrameDatabase(V, nkf, nkf * WPK + 10 * WPK)
        t0 = time.perf_counter()
        for k in range(nkf):
            db.add(k, *bows[k])
        t_add = (time.perf_counter() - t0) / nkf
        lists = {k: [j for j in (k - 1, k + 1, k - 2, k + 2, k - 3, k + 3, k - 4, k + 4, k - 5, k + 5) if 0 <= j < nkf] for k in range(nkf)}
        db.set_covisibles(lists)
        queries = [bow_at(shift * int(rng.integers(0, nkf)) + 7) for _ in range(32)]
        t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dt)).to(dev)
        dq = [(t(q[0], np.int32), t(q[1], np.float64), len(q[0])) for q in queries]
        d_conn = t(np.arange(10), np.int32)
        d_cand, d_n = torch.zeros(nkf, dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        res = {"keyframes": nkf, "postings": db.size()[1], "add_ms": round(t_add * 1e3, 4)}
        for mode, tag in ((0, "loop_query_ms"), (1, "reloc_query_ms")):
            def run():
                for qi, qv, nq in dq:
                    db.detect_device(mode, nq, qi.data_ptr(), qv.data_ptr(), 10, d_conn.data_ptr(), 0.0, nkf, d_cand.data_ptr(), d_n.data_ptr(),
                                     0, 0, stream.cuda_stream)
            for _ in range(args.warmup):
                run()
            stream.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(args.iters):
                run()
            e1.record(stream)
            stream.synchronize()
            res[tag] = round(e0.elapsed_time(e1) / (args.iters * len(dq)), 4)
        res["candidates_last_query"] = int(d_n.item())
        # erase + re-add of 100 keyframes
        t0 = time.perf_counter()
        for k in range(100):
            db.erase(k)
        res["erase_ms"] = round((time.perf_counter() - t0) / 100 * 1e3, 4)
        for k in range(100):
            db.add(k, *bows[k])
        # the stateless call on the same data: every keyframe's BowVector and covisibility list passed per query
        kf_ptr = np.cumsum([0] + [len(b[0]) for b in bows]).astype(np.int32)
        db_ids, db_vals = np.concatenate([b[0] for b in bows]), np.concatenate([b[1] for b in bows])
        cv_ptr = np.cumsum([0] + [len(lists[k]) for k in range(nkf)]).astype(np.int32)
        cv = np.concatenate([np.array(lists[k], np.int32) for k in range(nkf)])
        connected = np.zeros(nkf, np.uint8)
        connected[:10] = 1
        for mode, tag in ((0, "stateless_loop_wall_ms"), (1, "stateless_reloc_wall_ms")):
            BW.db_detect(m, mode, *queries[0], kf_ptr, db_ids, db_vals, connected, cv_ptr, cv)
            t0 = time.perf_counter()
            for q in queries[:8]:
                BW.db_detect(m, mode, *q, kf_ptr, db_ids, db_vals, connected, cv_ptr, cv)
            res[tag] = round((time.perf_counter() - t0) / 8 * 1e3, 4)
        out["%dk" % (nkf // 1000)] = res
        db.close()
    m.close()
    V.close()
    return out


def bowchain(args):
    """The BowVector built on the device (orbfe_bow_vector_device) and the relocalisation chain it completes, on 1920x1080
    frames of 2000 keypoints with a k = 10, L = 6 vocabulary (TF-IDF, L1), levelsup 4:
      bow_vector_{1,33}_frames_ms   CUDA-event ms of orbfe_bow_vector_device alone;
      chain_{device,host}_wall_ms   one extracted frame (descriptors in HBM) to SearchByBoW results against a resident database
                                    of 1000 keyframes (32 views of the place, added by orbfe_kfdb_add_device, and 968 unrelated
                                    ones).  Device: descent, BowVector, FeatureVector, detect_device on the padded row, one
                                    readback of the candidate count, search_by_bow_device.  Host: the path through the
                                    host-array transform -- descent and FeatureVector on the device, descriptors D2H,
                                    orbfe_bow_transform, BowVector H2D, detect_device, the same search;
      detect_{padded,exact}_ms      CUDA-event ms of detect_device on frame 0's row with nq = cap and with nq = its word count."""
    import torch
    import orb_slam_b200 as fe
    from orb_slam_b200 import matching as M, bow as BW
    from orb_slam_b200.synth import textured_frame, shifted_frame, random_vocabulary
    W, H, NF, levelsup, NREAL, NKF = 1920, 1080, 2000, 4, 32, 1000
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    s = stream.cuda_stream
    base = textured_frame(W, H, seed=21)
    # frame 0: the current frame; frames 1..32: keyframes of the same place
    frames = np.stack([base] + [shifted_frame(base, 4 * (i % 5) - 8, 3 * (i % 3) - 3, seed=i) for i in range(1, NREAL + 1)])
    F = len(frames)
    voc = random_vocabulary(10, 6, seed=3)
    V = BW.Vocabulary(voc)
    ex = fe.ORBextractor(NF, 1.2, 8)
    m = fe.ORBmatcher(0.75, True)
    i32 = lambda *shape: torch.zeros(shape, dtype=torch.int32, device=dev)
    d_frames = torch.from_numpy(frames).to(dev)
    # the frame store has a frame per database slot (slot = frame index); the unrelated keyframes' frames are empty
    d_kps = torch.zeros((NKF, NF, 28), dtype=torch.uint8, device=dev)
    d_desc = torch.zeros((NKF, NF, 32), dtype=torch.uint8, device=dev)
    d_valid = torch.ones((NKF, NF), dtype=torch.uint8, device=dev)
    d_cnt, d_leaf, d_node = i32(NKF), i32(F * NF), i32(F * NF)
    d_fid, d_fptr, d_fitems, d_fn = i32(NKF, NF), i32(NKF, NF + 1), i32(NKF, NF), i32(NKF)
    d_bid, d_bn = i32(F, NF), i32(F)
    d_bval = torch.zeros((F, NF), dtype=torch.float64, device=dev)
    d_cand, d_nc, d_zero = i32(NKF), i32(1), i32(NKF)
    d_out, d_nm = i32(NKF, NF), i32(NKF)
    torch.cuda.synchronize()
    ex.extract_batch_device(d_frames.data_ptr(), W, H, W, W * H, F, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), s)
    V.descend_device(d_desc.data_ptr(), F * NF, levelsup, d_leaf.data_ptr(), d_node.data_ptr(), s)
    bowv = lambda nf: BW.bow_vector_device(V, nf, d_leaf.data_ptr(), d_cnt.data_ptr(), NF, d_bid.data_ptr(), d_bval.data_ptr(),
                                           d_bn.data_ptr(), s)
    fvec = lambda nf: BW.feature_vector_device(V, nf, d_leaf.data_ptr(), d_node.data_ptr(), d_cnt.data_ptr(), NF, d_fid.data_ptr(),
                                               d_fptr.data_ptr(), d_fitems.data_ptr(), d_fn.data_ptr(), s)
    bowv(F)
    fvec(F)
    stream.synchronize()

    def timed(fn, iters=args.iters * 4, warm=args.warmup):
        for _ in range(warm):
            fn()
        stream.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(iters):
            fn()
        e1.record(stream)
        stream.synchronize()
        return e0.elapsed_time(e1) / iters

    out = {"what": "BowVector on the device and the relocalisation chain, 1920x1080 frames, %d keypoints, vocabulary k=10 L=6 "
                   "TF-IDF L1, levelsup %d, %d keyframes in the database" % (NF, levelsup, NKF), "counts_min": int(d_cnt[:F].min().item())}
    _gpu_and_power_limit(out)
    out["bow_vector_1_frame_ms"] = timed(lambda: bowv(1), iters=200)
    out["bow_vector_%d_frames_ms" % F] = timed(lambda: bowv(F), iters=200)
    out["words_per_frame_mean"] = float(d_bn.float().mean().item())
    # the sequential norm: the same launch on a vocabulary without a norm (TF, values divided by the word count)
    Vt = BW.Vocabulary(voc, BW.TF, BW.NORM_NONE)
    out["bow_vector_%d_frames_no_norm_ms" % F] = timed(lambda: BW.bow_vector_device(Vt, F, d_leaf.data_ptr(), d_cnt.data_ptr(), NF, d_bid.data_ptr(),
                                                                                   d_bval.data_ptr(), d_bn.data_ptr(), s), iters=200)
    Vt.close()

    # the database: 968 unrelated keyframes (host adds of random BowVectors), then the 32 views of the place from the device rows
    db = BW.KeyFrameDatabase(V, NKF, NKF * NF)
    rng = np.random.default_rng(7)
    nwords = int((voc["word_id"] >= 0).sum())
    for k in range(NREAL + 1, NKF):
        ids = np.unique(rng.integers(0, nwords, 1500)).astype(np.int32)
        v = rng.uniform(0.2, 3.0, len(ids))
        db.add(k, ids, v / v.sum())
    bowv(F)
    db.add_device(np.arange(1, NREAL + 1), np.arange(1, NREAL + 1), NF, d_bid.data_ptr(), d_bval.data_ptr(), d_bn.data_ptr(), s)
    db.set_covisibles({k: [j for j in (k - 1, k + 1, k - 2, k + 2) if 1 <= j <= NREAL] for k in range(1, NREAL + 1)})
    detect = lambda nq, qi, qv: db.detect_device(1, nq, qi, qv, 0, 0, 0.0, NKF, d_cand.data_ptr(), d_nc.data_ptr(), 0, 0, s)

    def search(nc):
        M.search_by_bow_device(m, 0, nc, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), NF, d_fid.data_ptr(), d_fptr.data_ptr(),
                               d_fitems.data_ptr(), d_fn.data_ptr(), d_valid.data_ptr(), d_cand.data_ptr(), d_zero.data_ptr(),
                               d_out.data_ptr(), d_nm.data_ptr(), s)
        stream.synchronize()

    def chain_device():
        V.descend_device(d_desc.data_ptr(), NF, levelsup, d_leaf.data_ptr(), d_node.data_ptr(), s)
        bowv(1)
        fvec(1)
        detect(NF, d_bid.data_ptr(), d_bval.data_ptr())
        nc = int(d_nc.item())
        search(nc)
        return nc

    def chain_host():
        V.descend_device(d_desc.data_ptr(), NF, levelsup, d_leaf.data_ptr(), d_node.data_ptr(), s)
        fvec(1)
        n0 = int(d_cnt[0].item())
        (ids, vals), _ = V.transform(d_desc[0, :n0].cpu().numpy(), levelsup)
        d_qi, d_qv = torch.from_numpy(ids).to(dev), torch.from_numpy(vals).to(dev)
        detect(len(ids), d_qi.data_ptr(), d_qv.data_ptr())
        nc = int(d_nc.item())
        search(nc)
        return nc, ids, vals

    with torch.cuda.stream(stream):
        # the two chains alternate, so that both see the same share of the host
        chains = (("device", chain_device), ("host", chain_host))
        lat = {tag: [] for tag, _ in chains}
        for it in range(args.warmup + args.iters * 20):
            for tag, fn in chains:
                t0 = time.perf_counter()
                fn()
                if it >= args.warmup:
                    lat[tag].append((time.perf_counter() - t0) * 1e3)
        results = {}
        for tag, fn in chains:
            out["chain_%s_wall_ms" % tag] = float(np.median(lat[tag]))
            out["chain_%s_wall_ms_p10_p90" % tag] = [float(np.percentile(lat[tag], 10)), float(np.percentile(lat[tag], 90))]
            r = fn()
            nc = r if tag == "device" else r[0]
            results[tag] = (d_cand[:nc].cpu().numpy(), d_nm[:nc].cpu().numpy(), d_out[:nc].cpu().numpy())
            if tag == "host":
                ids, vals = r[1], r[2]
        m.sync()
        chain_device()
        n0 = int(d_bn[0].item())
        out["same_bow_vector"] = bool(np.array_equal(d_bid[0, :n0].cpu().numpy(), ids) and
                                      np.array_equal(d_bval[0, :n0].cpu().numpy().view(np.uint64), vals.view(np.uint64)))
    (cd, nd, od), (ch, nh, oh) = results["device"], results["host"]
    out["candidates"] = cd.tolist()
    out["matches"] = int(nd.sum())
    out["same_as_host_chain"] = bool(np.array_equal(cd, ch) and np.array_equal(nd, nh) and np.array_equal(od, oh))
    # padded and exact alternate over several windows of 100 queries each: the spread of each is reported beside it
    det = {"padded": [], "exact": []}
    for _ in range(6):
        det["padded"].append(timed(lambda: detect(NF, d_bid.data_ptr(), d_bval.data_ptr()), iters=100))
        det["exact"].append(timed(lambda: detect(n0, d_bid.data_ptr(), d_bval.data_ptr()), iters=100))
    for tag, v in det.items():
        out["detect_%s_ms" % tag] = float(np.median(v))
        out["detect_%s_ms_min_max" % tag] = [float(min(v)), float(max(v))]
    out["words_frame0"] = n0
    db.close(); ex.close(); V.close(); m.close()
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--what", default="config3,config5")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--groups", type=int, default=10000)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    for w in args.what.split(","):
        print(json.dumps({"config3": config3, "config5": config5, "small": small, "exchange1": exchange1, "matchers": matchers, "h2d": h2d, "fast": fast, "latency": latency,
                          "reloc": reloc, "mapping": mapping, "mapdesc": mapdesc, "kfdb": kfdb, "bowchain": bowchain,
                          "windowed": windowed}[w](args)))
