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
  --what kfdbbatch the same databases: CUDA-event ms of orbfe_kfdb_detect_batch_device for B = 1, 8, 32, 64 relocalisation
                   queries (and 64 loop queries at 1k) against B consecutive orbfe_kfdb_detect_device calls, outputs compared;
                   --baseline-lib PATH alternates the single-query detect_device of another build with this one's
  --what bowchain  the BowVector kernel alone for 1 and 33 1080p / 2000-keypoint frames (CUDA events), relocalisation from an
                   extracted frame to SearchByBoW results against a resident 1000-keyframe database with the BowVector built
                   on the device vs on the host (wall time), and detect_device on a padded row vs its word count
  --what windowed  wall time per call of the host-array windowed matchers (staging, launch, copy back, synchronise):
                   orbfe_search_by_projection_frames for 1 and 8 pairs, orbfe_search_local_points and orbfe_window_search at
                   1080p / 2000 keypoints, orbfe_search_for_initialization at 720p / 2000 keypoints
  --what guided    wall time per call of orbfe_guided_best and orbfe_guided_search (rule 0, no histogram) for 1000, 5000 and
                   30000 Fuse / SearchBySim3 windows on one 1080p / 2000-keypoint keyframe; --baseline-lib PATH alternates
                   every call with another build of liborbfe.so in the same process and compares the outputs

  --what loopscore LoopClosing::DetectLoop's minScore on the device (orbfe_bow_min_score_device): CUDA-event us per call for 1 query
                   x 30 and x 100 connected keyframes and 16 queries x 30, rows of ~1000 and ~2000 words, against the host path
                   (rows D2H, CPU score, one float H2D) and, with --baseline-lib, the same entry of another build alternately.
  --what vocload   orbfe_vocabulary_load_text on a synthetic ORBvoc-shaped text (k = 10, L = 6: 1,111,111 lines, internal nodes
                   weighted 0, words with 6 significant digits like Data/ORBvoc.txt) and on the same tree with %r weights (the
                   host-conversion path): wall time per load (file read included), device time per kernel and copy
                   (torch.profiler, a run of its own), and the reference's loadFromTextFile from oracle/_ref in the same process.
  --what normaldepth MapPoint::UpdateNormalAndDepth after LocalBundleAdjustment (Optimizer.cc:488): every local map point of
                   20 local keyframes of 2000 features (10000 points, 2-60 observations, over a 60-keyframe store) after
                   SetWorldPos, in one batch: CUDA-event ms of orbfe_normal_and_depth_device, the wall time of
                   orbfe_normal_and_depth including the host gather of the centres and its staging, and the wall time of the
                   oracle's C loop on the same arrays (plain float / double C, not OpenCV's cv::Mat), outputs compared.
  --what covis     KeyFrame::UpdateConnections on the resident covisibility graph (orbfe_covis_update_connections_device) of a
                   2000-keyframe map (2000 features each, ~8 observations per point, tests/covis_scenes.py scene_large), after
                   every keyframe was updated once: CUDA-event ms of a batch of 1 (LocalMapping's call) and of a batch of 64
                   (loop correction), and the wall time of the oracle's C restatement (oracle/orb_oracle_covis.c: dense rows, not
                   the reference's std::map) for the same calls.
  --what observations MapPoint::GetObservations() built on the device from the keyframes' rows
                   (orbfe_covis_observations_device) on the same 2000-keyframe map: CUDA-event ms for the points of one
                   keyframe's row (ProcessNewKeyFrame) and for every point of the map, and the wall time of the host build
                   of the same lists from the reference's own MapPoints (GetObservations() copied, walked and flattened;
                   the upload not included), lists compared.
  --what kfculling LocalMapping::KeyFrameCulling on the device (orbfe_covis_keyframe_culling_device) on 2000-keyframe maps of
                   2000 features (tests/covis_scenes.py scene_large with points spread over +-5, +-25 and +-64 keyframes, so the
                   current keyframe has about 20, 100 and up to 256 = max_connections covisible keyframes): CUDA-event ms of one call
                   with culls allowed at the front of the list, in its middle and nowhere (mbNotErase on the others), each from
                   the same state; the wall time of the C oracle for the same calls (verdicts compared); and the wall time of the
                   reference's own KeyFrameCulling() on the same map with culls nowhere.
  --what localmap  Tracking::UpdateReference on the device (orbfe_covis_local_map_device) on the 2000-keyframe x 2000-feature map
                   of tests/covis_scenes.py scene_large, for frames of about 300, 1000 and 2000 matched points
                   (tests/local_map_scenes.py large_frames): the median of CUDA-event windows of one call each, and the wall
                   time of the reference's own UpdateReference() on the same map with the same lists (results compared).
  --what multigeom  a three-camera rig step (one 1920x1080 and two 1280x720 cameras, 2000 kp, 8 levels) at 1 and 4 frames per
                   camera: CUDA-event ms and wall ms per step of one orbfe_extract_multi_device call, of three handles one after
                   another on one stream and of three handles on three streams (forked from and joined to one stream by events).
                   The three ways run alternately, five rounds of 200 steps each; the median round is reported.
  --what multitrack the matching half of that rig step: frame-to-frame SearchByProjection for every camera of the --what
                   multigeom rig (frames extracted in one orbfe_extract_multi_device call) at 1 and 4 pairs per camera:
                   CUDA-event ms and wall ms per step of one orbfe_search_by_projection_cams_device call, of three
                   single-geometry calls one after another on one stream and of three calls on three streams (three matcher
                   handles, forked from and joined to one stream by events).  Every step first resets the Current frames'
                   slots (one fill on the main stream, in all three ways).  Alternating rounds as --what multigeom; the
                   outputs of the three ways are compared.
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


def guided(args):
    """orbfe_guided_best and orbfe_guided_search (rule 0, no histogram) one call at a time, as the facade's Fuse,
    SearchBySim3 and SearchByProjection(KeyFrame*, Scw, ...) call them: median wall ms per call (staging, launch, copy back,
    synchronise) for 1000, 5000 and 30000 windows on one extracted 1920x1080 keyframe of 2000 features.  Windows are map
    points seen from a nearby pose: centred near a feature, radius th = 3 times the scale factor of the predicted level,
    levels [lv - 1, lv].  With --baseline-lib the same calls alternate with that build of liborbfe.so in one process, and
    same_as_baseline compares every output (a refused call is recorded as null)."""
    import orb_slam_b200 as fe
    from orb_slam_b200 import matching as M
    from orb_slam_b200.synth import noisy_copies, textured_frame
    NF, W, H = 2000, 1920, 1080
    ex = fe.ORBextractor(NF, 1.2, 8)
    kps, desc, cnt = ex.extract_batch(textured_frame(W, H, seed=9)[None])
    ex.close()
    k, d = kps[0, :cnt[0]], desc[0, :cnt[0]]
    view = M.FrameView(k, d, W, H)
    vp = C.c_void_p
    libs = {"this": fe.lib()}
    if args.baseline_lib:
        libs["baseline"] = C.CDLL(os.path.abspath(args.baseline_lib))
    handles = {}
    for name, L in libs.items():
        L.orbfe_matcher_create.argtypes = [C.c_int, C.POINTER(vp)]
        L.orbfe_matcher_destroy.argtypes = [vp]
        L.orbfe_guided_best.argtypes = [vp, vp, C.c_int] + [vp] * 6 + [C.c_int, vp]
        L.orbfe_guided_search.argtypes = [vp, vp, C.c_int] + [vp] * 7 + [C.c_int, C.c_float, C.c_int, C.c_int, vp, vp]
        h = vp()
        assert L.orbfe_matcher_create(0, C.byref(h)) == 0, name
        handles[name] = h
    p = lambda a: a.ctypes.data_as(vp)
    rng = np.random.default_rng(5)
    out = {"what": "guided_best / guided_search (rule 0, hist 0) wall ms per call, 1920x1080 keyframe, %d features" % len(k),
           "baseline": args.baseline_lib or None}
    same = True
    for nq in (1000, 5000, 30000):
        src = rng.integers(0, len(k), nq)
        lv = np.clip(k["octave"][src].astype(np.int32) + rng.integers(-1, 2, nq), 0, 7).astype(np.int32)
        qu = (k["x"][src] + rng.normal(0, 1.5, nq)).astype(np.float32)
        qv = (k["y"][src] + rng.normal(0, 1.5, nq)).astype(np.float32)
        qr = (np.float32(3.0) * view.sf[lv]).astype(np.float32)
        lo, hi = (lv - 1).astype(np.int32), lv
        qd = noisy_copies(d[src], 0.1, 6)
        res = {}

        def best(name):
            o = np.full(nq, -1, np.int32)
            rc = libs[name].orbfe_guided_best(handles[name], C.byref(view.c), nq, p(qu), p(qv), p(qr), p(lo), p(hi), p(qd), 50, p(o))
            return o if rc == 0 else None

        def search(name):
            so, nm = np.full(len(k), -1, np.int32), C.c_int(0)
            rc = libs[name].orbfe_guided_search(handles[name], C.byref(view.c), nq, p(qu), p(qv), p(qr), p(lo), p(hi), p(qd), None,
                                                0, 0.0, 50, 0, p(so), C.byref(nm))
            return (nm.value, so) if rc == 0 else None
        for fn_name, fn in (("best", best), ("search", search)):
            for name in libs:
                for _ in range(args.warmup):
                    res[(fn_name, name)] = fn(name)
            lat = {name: [] for name in libs}
            order = list(libs)
            for it in range(args.iters * 20):
                for name in (order if it % 2 == 0 else order[::-1]):   # alternate which build goes first
                    t0 = time.perf_counter()
                    fn(name)
                    lat[name].append((time.perf_counter() - t0) * 1e3)
            for name in libs:
                r = res[(fn_name, name)]
                out["%s_%d_%s_wall_ms" % (fn_name, nq, name)] = float(np.median(lat[name])) if r is not None else None
            r0 = res[(fn_name, "this")]
            out["%s_%d_kept" % (fn_name, nq)] = int((r0 >= 0).sum()) if fn_name == "best" else r0[0]
            if "baseline" in libs and res[(fn_name, "baseline")] is not None:
                rb = res[(fn_name, "baseline")]
                same &= bool(np.array_equal(r0, rb)) if fn_name == "best" else (r0[0] == rb[0] and bool(np.array_equal(r0[1], rb[1])))
    out["same_as_baseline"] = same if "baseline" in libs else None
    for name, L in libs.items():
        L.orbfe_matcher_destroy(handles[name])
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


def multigeom(args):
    """See the module docstring (--what multigeom)."""
    import torch
    import orb_slam_b200 as fe
    from orb_slam_b200.synth import textured_frame
    dev = torch.device("cuda", 0)
    cams = [(1920, 1080), (1280, 720), (1280, 720)]
    NF, steps, rounds = 2000, 200, 5
    main = torch.cuda.Stream(device=dev)
    side = [torch.cuda.Stream(device=dev) for _ in cams]
    out = {"what": "rig step of 1x1920x1080 + 2x1280x720 cameras, %d kp, 8 levels, device-resident: ms per step (median of %d rounds "
                   "of %d steps)" % (NF, rounds, steps)}
    for B in (1, 4):
        frames = [torch.from_numpy(np.stack([textured_frame(W, H, seed=10 * c + i) for i in range(B)])).to(dev)
                  for c, (W, H) in enumerate(cams)]
        F = B * len(cams)
        multi = fe.ORBextractor(NF, 1.2, 8, fe.FAST_SCORE, 20)
        singles = [fe.ORBextractor(NF, 1.2, 8, fe.FAST_SCORE, 20) for _ in cams]
        slots = int(multi.tables()[2].sum())
        d_kps = torch.empty((F, slots, 28), dtype=torch.uint8, device=dev)
        d_desc = torch.empty((F, slots, 32), dtype=torch.uint8, device=dev)
        d_cnt = torch.empty((F,), dtype=torch.int32, device=dev)
        groups = [(f.data_ptr(), W, H, W, W * H, B) for f, (W, H) in zip(frames, cams)]

        def run_multi():
            multi.extract_multi_device(groups, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), main.cuda_stream)

        def run_serial(streams=None):
            for c, (ex, (p, W, H, st, fs, b)) in enumerate(zip(singles, groups)):
                s = streams[c] if streams else main
                ex.extract_batch_device(p, W, H, st, fs, b, d_kps[c * B].data_ptr(), d_desc[c * B].data_ptr(), d_cnt[c * B].data_ptr(),
                                        s.cuda_stream)

        def run_streams():
            fork = torch.cuda.Event()
            fork.record(main)
            for s in side:
                s.wait_event(fork)
            run_serial(side)
            for s in side:
                ev = torch.cuda.Event()
                ev.record(s)
                main.wait_event(ev)

        ways = {"multi_one_call": run_multi, "three_handles_one_stream": run_serial, "three_handles_three_streams": run_streams}
        res = {k: {"event_ms": [], "wall_ms": []} for k in ways}
        for fn in ways.values():
            for _ in range(max(args.warmup, 10)):
                fn()
        torch.cuda.synchronize()
        want = None
        for r in range(rounds):
            for name, fn in ways.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                e0.record(main)
                for _ in range(steps):
                    fn()
                e1.record(main)
                e1.synchronize()
                torch.cuda.synchronize()
                res[name]["wall_ms"].append((time.perf_counter() - t0) * 1e3 / steps)
                res[name]["event_ms"].append(e0.elapsed_time(e1) / steps)
                got = (d_cnt.cpu().numpy().tolist(), int(d_desc.sum().item()))
                want = want or got
                res[name]["same_outputs"] = res[name].get("same_outputs", True) and got == want
        out["%d_frame_per_camera" % B] = {k: {"event_ms": round(float(np.median(v["event_ms"])), 4),
                                              "wall_ms": round(float(np.median(v["wall_ms"])), 4),
                                              "event_ms_min_max": [round(min(v["event_ms"]), 4), round(max(v["event_ms"]), 4)],
                                              "same_outputs": v["same_outputs"]} for k, v in res.items()}
        out["%d_frame_per_camera" % B]["multi_launches"] = multi.last_launches()
        multi.close()
        for ex in singles:
            ex.close()
    _gpu_and_power_limit(out)
    try:
        import subprocess
        out["sm_clock"] = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                                         capture_output=True, text=True).stdout.strip()
    except Exception as e:
        out["sm_clock"] = "unknown: %r" % e
    return out


def multitrack(args):
    """See the module docstring (--what multitrack)."""
    import torch
    import orb_slam_b200 as fe
    from orb_slam_b200 import matching as M
    from orb_slam_b200.synth import textured_frame
    dev = torch.device("cuda", 0)
    cams = [(1920, 1080), (1280, 720), (1280, 720)]
    NF, steps, rounds, TH = 2000, 200, 5, 7.0
    main = torch.cuda.Stream(device=dev)
    side = [torch.cuda.Stream(device=dev) for _ in cams]
    table = [(0.0, 0.0, float(W), float(H), 0.7 * W, 0.7 * W, W / 2, H / 2) for W, H in cams]
    out = {"what": "rig SearchByProjection(Frame, Frame) of 1x1920x1080 + 2x1280x720 cameras, %d kp, 8 levels, device-resident: ms "
                   "per step (median of %d rounds of %d steps)" % (NF, rounds, steps)}
    for B in (1, 4):
        # B + 1 frames per camera, each shifted by (3, 2) px from the one before; pair i of a camera = (frame i + 1, frame i)
        frames = []
        for c, (W, H) in enumerate(cams):
            base = textured_frame(W + 3 * B + 3, H + 2 * B + 2, seed=20 + c)
            frames.append(torch.from_numpy(np.stack([np.ascontiguousarray(base[2 * i:2 * i + H, 3 * i:3 * i + W])
                                                     for i in range(B + 1)])).to(dev))
        F, P = (B + 1) * len(cams), B * len(cams)
        ex = fe.ORBextractor(NF, 1.2, 8, fe.FAST_SCORE, 20)
        cap = int(ex.tables()[2].sum())
        d_kps = torch.empty((F, cap, 28), dtype=torch.uint8, device=dev)
        d_desc = torch.empty((F, cap, 32), dtype=torch.uint8, device=dev)
        d_cnt = torch.empty((F,), dtype=torch.int32, device=dev)
        ex.extract_multi_device([(f.data_ptr(), W, H, W, W * H, B + 1) for f, (W, H) in zip(frames, cams)], d_kps.data_ptr(),
                                d_desc.data_ptr(), d_cnt.data_ptr())
        ex.sync()
        torch.cuda.synchronize()
        ex.close()
        kps = d_kps.cpu().numpy().view(fe.KP_DTYPE).reshape(F, cap)
        cnt = d_cnt.cpu().numpy()
        world = np.zeros((F, cap, 3), np.float32)
        flags = np.zeros((F, cap), np.uint8)
        frame_cam = np.repeat(np.arange(len(cams), dtype=np.int32), B + 1)
        for f in range(F):
            _, _, _, _, fx, fy, cx, cy = table[frame_cam[f]]
            k = kps[f, :cnt[f]]
            world[f, :cnt[f], 0] = (k["x"] - np.float32(cx)) / np.float32(fx) * np.float32(4)
            world[f, :cnt[f], 1] = (k["y"] - np.float32(cy)) / np.float32(fy) * np.float32(4)
            world[f, :cnt[f], 2] = 4
            flags[f, :cnt[f]] = 1
        cur = np.array([c * (B + 1) + i + 1 for c in range(len(cams)) for i in range(B)], np.int32)
        Tcw = np.zeros((P, 12), np.float32)
        for j, f in enumerate(cur):
            fx = np.float32(table[frame_cam[f]][4])
            Tcw[j] = [1, 0, 0, -12 / fx, 0, 1, 0, -8 / fx, 0, 0, 1, 0.01]
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        d_cur, d_last, d_world, d_flags, d_T, d_fc = t(cur), t(cur - 1), t(world), t(flags), t(Tcw), t(frame_cam)
        d_mp = torch.full((P, cap), -1, dtype=torch.int32, device=dev)
        d_nm = torch.zeros((P,), dtype=torch.int32, device=dev)
        store = [d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr()]
        multi = fe.ORBmatcher(0.9, True)
        singles = [fe.ORBmatcher(0.9, True) for _ in cams]
        L = M._bind()
        vp = C.c_void_p

        def reset():
            with torch.cuda.stream(main):
                d_mp.fill_(-1)

        def run_multi():
            reset()
            M.search_by_projection_cams_device(multi, P, *store, cap, d_cur.data_ptr(), d_last.data_ptr(), d_world.data_ptr(),
                                               d_flags.data_ptr(), d_T.data_ptr(), table, d_fc.data_ptr(), 1.2, 8, TH,
                                               d_mp.data_ptr(), d_nm.data_ptr(), main.cuda_stream)

        def run_serial(streams=None):
            if streams is None:
                reset()
            for c, cam in enumerate(table):
                x0, y0, x1, y1, fx, fy, cx, cy = cam
                s = streams[c] if streams else main
                m = singles[c]
                rc = L.orbfe_search_by_projection_device(m.handle, B, *[vp(p) for p in store], cap, vp(d_cur[c * B].data_ptr()),
                                                         vp(d_last[c * B].data_ptr()), vp(d_world.data_ptr()), vp(d_flags.data_ptr()),
                                                         vp(d_T[c * B].data_ptr()), x0, y0, x1, y1, 1.2, 8, fx, fy, cx, cy, TH, 1,
                                                         vp(d_mp[c * B].data_ptr()), vp(d_nm[c * B:].data_ptr()), vp(s.cuda_stream))
                assert rc == 0, L.orbfe_last_error()

        def run_streams():
            reset()
            fork = torch.cuda.Event()
            fork.record(main)
            for s in side:
                s.wait_event(fork)
            run_serial(side)
            for s in side:
                ev = torch.cuda.Event()
                ev.record(s)
                main.wait_event(ev)

        ways = {"cams_one_call": run_multi, "three_calls_one_stream": run_serial, "three_calls_three_streams": run_streams}
        res = {k: {"event_ms": [], "wall_ms": []} for k in ways}
        for fn in ways.values():
            for _ in range(max(args.warmup, 10)):
                fn()
        torch.cuda.synchronize()
        want = None
        for r in range(rounds):
            for name, fn in ways.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                e0.record(main)
                for _ in range(steps):
                    fn()
                e1.record(main)
                e1.synchronize()
                torch.cuda.synchronize()
                res[name]["wall_ms"].append((time.perf_counter() - t0) * 1e3 / steps)
                res[name]["event_ms"].append(e0.elapsed_time(e1) / steps)
                got = (d_nm.cpu().numpy().tolist(), d_mp.cpu().numpy().tobytes())
                want = want or got
                res[name]["same_outputs"] = res[name].get("same_outputs", True) and got == want
        for m in [multi] + singles:
            m.sync()
        out["%d_pair_per_camera" % B] = {k: {"event_ms": round(float(np.median(v["event_ms"])), 4),
                                             "wall_ms": round(float(np.median(v["wall_ms"])), 4),
                                             "event_ms_min_max": [round(min(v["event_ms"]), 4), round(max(v["event_ms"]), 4)],
                                             "same_outputs": v["same_outputs"]} for k, v in res.items()}
        out["%d_pair_per_camera" % B]["nmatches"] = want[0]
        multi.close()
        for m in singles:
            m.close()
    _gpu_and_power_limit(out)
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


def kfdbbatch(args):
    """orbfe_kfdb_detect_batch_device against B consecutive orbfe_kfdb_detect_device calls on one stream (CUDA events, outputs
    compared), on the databases of --what kfdb (1k and 10k keyframes of about 1000 words, ids over 10^6): B = 1, 8, 32, 64
    relocalisation queries as padded rows of 2048 entries (about 2000 words each), and one loop-mode line at 1k.  With
    --baseline-lib, the single-query orbfe_kfdb_detect_device of that build and of this one alternate in one process on
    twin databases (median of repeated CUDA-event windows of 32 queries each)."""
    import torch
    NW, WPK, QW, QCAP = 1_000_000, 1000, 2000, 2048
    n = NW + 1
    cp = np.zeros(n + 1, np.int32)
    cp[1:] = NW
    voc = {"node_desc": np.zeros((n, 32), np.uint8), "child_ptr": cp, "children": np.arange(1, n, dtype=np.int32),
           "word_id": np.arange(-1, NW, dtype=np.int32), "weight": np.ones(n)}
    vp, i_, p = C.c_void_p, C.c_int, (lambda a: a.ctypes.data_as(C.c_void_p))
    import orb_slam_b200 as fe
    libs = {"this": fe.lib()}
    if args.baseline_lib:
        libs["baseline"] = C.CDLL(os.path.abspath(args.baseline_lib))
    for L in libs.values():
        L.orbfe_vocabulary_create.argtypes = [i_, i_, i_, vp, vp, vp, vp, vp, i_, i_]
        L.orbfe_vocabulary_create.restype = vp
        L.orbfe_vocabulary_destroy.argtypes = [vp]
        L.orbfe_kfdb_create.argtypes = [vp, i_, C.c_longlong, C.POINTER(vp)]
        L.orbfe_kfdb_destroy.argtypes = [vp]
        L.orbfe_kfdb_add.argtypes = [vp, i_, i_, vp, vp]
        L.orbfe_kfdb_set_covisibles.argtypes = [vp, i_, vp, vp, vp]
        L.orbfe_kfdb_detect_device.argtypes = [vp, i_, i_, vp, vp, i_, vp, C.c_float, i_, vp, vp, vp, vp, vp]
    libs["this"].orbfe_kfdb_create_batched.argtypes = [vp, i_, C.c_longlong, i_, C.POINTER(vp)]
    libs["this"].orbfe_kfdb_detect_batch_device.argtypes = [vp, i_, i_, i_, vp, vp, vp, vp, vp, i_, vp, vp, vp, vp, vp]
    vocs = {name: L.orbfe_vocabulary_create(0, n, 1, p(voc["node_desc"]), p(voc["child_ptr"]), p(voc["children"]), p(voc["word_id"]),
                                            p(voc["weight"]), 0, 1) for name, L in libs.items()}
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    out = {"what": "KeyFrameDatabase batched queries: CUDA-event ms per batch of B vs B consecutive detect_device calls; %d words per "
                   "keyframe, queries of about %d words as rows of %d, word ids over 10^6" % (WPK, QW, QCAP),
           "baseline": args.baseline_lib or None}
    _gpu_and_power_limit(out)
    try:
        import subprocess
        out["sm_clock"] = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                                         capture_output=True, text=True).stdout.strip()
    except Exception as e:
        out["sm_clock"] = "unknown: %r" % e
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dt)).to(dev)

    def events(fn, iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(iters):
            fn()
        e1.record(stream)
        stream.synchronize()
        return e0.elapsed_time(e1) / iters

    for nkf in (1000, 10000):
        rng = np.random.default_rng(nkf)
        shift = 100
        track = rng.integers(0, NW, nkf * shift + 4 * QW)

        def bow_at(pos, nw):
            w = track[pos:pos + nw].copy()
            flip = rng.random(nw) < 0.25
            w[flip] = rng.integers(0, NW, int(flip.sum()))
            ids = np.unique(w).astype(np.int32)
            v = rng.uniform(0.2, 3.0, len(ids))
            return ids, v / v.sum()

        bows = [bow_at(shift * k, WPK) for k in range(nkf)]
        lists = {k: [j for j in (k - 1, k + 1, k - 2, k + 2, k - 3, k + 3, k - 4, k + 4, k - 5, k + 5) if 0 <= j < nkf] for k in range(nkf)}
        slots = np.arange(nkf, dtype=np.int32)
        ptr = np.cumsum([0] + [len(lists[k]) for k in range(nkf)]).astype(np.int32)
        flat = np.concatenate([np.array(lists[k], np.int32) for k in range(nkf)])
        P = nkf * WPK + 10 * WPK

        def make(name, max_queries):
            L, h = libs[name], vp()
            rc = (L.orbfe_kfdb_create_batched(vocs[name], nkf, P, max_queries, C.byref(h)) if max_queries > 1 else
                  L.orbfe_kfdb_create(vocs[name], nkf, P, C.byref(h)))
            assert rc == 0, name
            for k in range(nkf):
                ids, vals = np.ascontiguousarray(bows[k][0]), np.ascontiguousarray(bows[k][1])
                assert L.orbfe_kfdb_add(h, k, len(ids), p(ids), p(vals)) == 0
            assert L.orbfe_kfdb_set_covisibles(h, nkf, p(slots), p(ptr), p(flat)) == 0
            return h

        queries = [bow_at(shift * int(rng.integers(0, nkf)) + 7, QW) for _ in range(64)]
        ids = np.full((64, QCAP), np.iinfo(np.int32).max, np.int32)
        vals = np.zeros((64, QCAP))
        for b, (qi, qv) in enumerate(queries):
            ids[b, :len(qi)], vals[b, :len(qi)] = qi, qv
        d_ids, d_vals = t(ids, np.int32), t(vals, np.float64)
        conn = np.arange(10, dtype=np.int32)
        d_conn, d_cptr = t(np.tile(conn, 64), np.int32), t(np.arange(65) * 10, np.int32)
        d_ms = t(np.full(64, 0.0), np.float32)
        res = {"keyframes": nkf, "query_words_mean": float(np.mean([len(q[0]) for q in queries]))}
        batched, seq = make("this", 64), make("this", 1)
        L = libs["this"]
        d_cand = [torch.zeros(64 * nkf, dtype=torch.int32, device=dev) for _ in range(2)]
        d_n = [torch.zeros(64, dtype=torch.int32, device=dev) for _ in range(2)]
        torch.cuda.synchronize()
        modes = [(1, B) for B in (1, 8, 32, 64)] + ([(0, 64)] if nkf == 1000 else [])
        for mode, Bq in modes:
            def run_batch():
                L.orbfe_kfdb_detect_batch_device(batched, mode, Bq, QCAP, d_ids.data_ptr(), d_vals.data_ptr(), d_cptr.data_ptr(), d_conn.data_ptr(),
                                                 d_ms.data_ptr(), nkf, d_cand[0].data_ptr(), d_n[0].data_ptr(), None, None, stream.cuda_stream)

            def run_seq():
                for b in range(Bq):
                    L.orbfe_kfdb_detect_device(seq, mode, QCAP, d_ids[b].data_ptr(), d_vals[b].data_ptr(), 10, d_conn.data_ptr(), 0.0, nkf,
                                               d_cand[1][b * nkf:].data_ptr(), d_n[1][b:].data_ptr(), None, None, stream.cuda_stream)
            # same outputs first (both databases have answered the same queries so far), then the timing
            run_batch()
            run_seq()
            stream.synchronize()
            n0, n1 = d_n[0][:Bq].cpu().numpy(), d_n[1][:Bq].cpu().numpy()
            c0, c1 = d_cand[0].cpu().numpy(), d_cand[1].cpu().numpy()
            same = bool(np.array_equal(n0, n1)) and all(np.array_equal(c0[b * nkf:b * nkf + n0[b]], c1[b * nkf:b * nkf + n0[b]]) for b in range(Bq))
            for _ in range(args.warmup):
                run_batch()
                run_seq()
            tb, ts = [], []
            for _ in range(5):
                tb.append(events(run_batch, args.iters))
                ts.append(events(run_seq, args.iters))
            tag = "%s_B%d" % ("loop" if mode == 0 else "reloc", Bq)
            res[tag] = {"batch_ms": round(float(np.median(tb)), 4), "sequential_ms": round(float(np.median(ts)), 4),
                        "batch_ms_min_max": [round(min(tb), 4), round(max(tb), 4)], "sequential_ms_min_max": [round(min(ts), 4), round(max(ts), 4)],
                        "speedup": round(float(np.median(ts) / np.median(tb)), 2), "same_outputs": same,
                        "candidates_mean": float(n0.mean())}
        L.orbfe_kfdb_destroy(batched)
        L.orbfe_kfdb_destroy(seq)
        # single-query regression: this build's detect_device and the baseline's, alternating, on twin databases
        if "baseline" in libs:
            hs = {name: make(name, 1) for name in libs}
            outs = {name: (torch.zeros(nkf, dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.int32, device=dev)) for name in libs}
            lat = {name: [] for name in libs}
            same = True
            for rep in range(args.iters * 4):
                for name in (list(libs) if rep % 2 == 0 else list(libs)[::-1]):
                    def run(name=name):
                        for b in range(32):
                            libs[name].orbfe_kfdb_detect_device(hs[name], 1, QCAP, d_ids[b].data_ptr(), d_vals[b].data_ptr(), 0, None, 0.0, nkf,
                                                                outs[name][0].data_ptr(), outs[name][1].data_ptr(), None, None, stream.cuda_stream)
                    lat[name].append(events(run, 1) / 32)
                c = {name: (outs[name][1].item(), outs[name][0][:outs[name][1].item()].cpu().numpy()) for name in libs}
                same &= c["this"][0] == c["baseline"][0] and bool(np.array_equal(c["this"][1], c["baseline"][1]))
            for name in libs:
                res["single_reloc_%s_ms" % name] = round(float(np.median(lat[name][2:])), 4)
                res["single_reloc_%s_ms_min_max" % name] = [round(min(lat[name][2:]), 4), round(max(lat[name][2:]), 4)]
                libs[name].orbfe_kfdb_destroy(hs[name])
            res["single_same_as_baseline"] = same
        out["%dk" % (nkf // 1000)] = res
    for name, L in libs.items():
        L.orbfe_vocabulary_destroy(vocs[name])
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


def loopscore(args):
    """LoopClosing::DetectLoop's minScore on the device (orbfe_bow_min_score_device) at its call site's shapes: 1 keyframe with
    30 and with 100 connected keyframes, and 16 queued keyframes with 30 each, on BowVector rows of about 1000 and about 2000
    words (word ids over 10^6, neighbouring rows sharing most words, as --what kfdb builds them).  CUDA-event microseconds per
    call over many launches on one stream after warm-up.  With --baseline-lib, the same entry of that build is timed
    alternately in the same process and its outputs compared bit for bit.  host_path_us is what a host without this entry
    does per keyframe, as wall time: one device gather of the rows and three D2H copies, L1Scoring::score on the CPU (the
    oracle's C restatement), H2D of the one float, one synchronise."""
    import torch
    from oracle import bow_score as OS
    NW = 1_000_000
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    vp, i_ = C.c_void_p, C.c_int
    libs = {"this": C.CDLL(os.path.join(ROOT, "orb_slam_b200", "liborbfe.so"))}
    if args.baseline_lib:
        libs["baseline"] = C.CDLL(args.baseline_lib)
    p = lambda a: a.ctypes.data_as(vp)
    vocs = {}
    for name, L in libs.items():
        L.orbfe_vocabulary_create.argtypes = [i_, i_, i_, vp, vp, vp, vp, vp, i_, i_]
        L.orbfe_vocabulary_create.restype = vp
        L.orbfe_vocabulary_destroy.argtypes = [vp]
        L.orbfe_vocabulary_destroy.restype = None
        L.orbfe_bow_min_score_device.argtypes = [vp, i_, i_, i_, vp, vp, vp, vp, vp, vp, vp, vp, vp]
        flat = (np.zeros((3, 32), np.uint8), np.array([0, 2, 2, 2], np.int32), np.array([1, 2], np.int32), np.array([-1, 0, 1], np.int32),
                np.ones(3))
        vocs[name] = L.orbfe_vocabulary_create(0, 3, 1, p(flat[0]), p(flat[1]), p(flat[2]), p(flat[3]), p(flat[4]), 0, 1)
        assert vocs[name]
    out = {"what": "minScore of LoopClosing::DetectLoop on device BowVector rows, word ids over 10^6; microseconds per call"}
    _gpu_and_power_limit(out)
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dt)).to(dev)
    F, reps = 128, 40 * args.iters
    for wpk in (1000, 2000):
        rng = np.random.default_rng(wpk)
        cap = 2 * wpk
        track = rng.integers(0, NW, F * wpk // 10 + 4 * wpk)
        ids = np.full((F, cap), 2 ** 31 - 1, np.int32)
        vals = np.zeros((F, cap))
        n = np.zeros(F, np.int32)
        for f in range(F):
            w = track[f * wpk // 10:f * wpk // 10 + wpk].copy()
            flip = rng.random(wpk) < 0.25
            w[flip] = rng.integers(0, NW, int(flip.sum()))
            u = np.unique(w).astype(np.int32)
            v = rng.uniform(0.2, 3.0, len(u))
            ids[f, :len(u)], vals[f, :len(u)], n[f] = u, v / v.sum(), len(u)
        d_ids, d_vals, d_n = t(ids, np.int32), t(vals, np.float64), t(n, np.int32)
        res = {"words_per_row": int(n.mean()), "cap": cap}
        for nq, ncov in ((1, 30), (1, 100), (16, 30)):
            qrow = (np.arange(nq) * 5 + 40).astype(np.int32)
            cov = np.concatenate([(q + np.array([(-1) ** j * (j // 2 + 1) for j in range(ncov)])) % F for q in qrow]).astype(np.int32)
            ptr = (np.arange(nq + 1) * ncov).astype(np.int32)
            d_q, d_ptr, d_cov = t(qrow, np.int32), t(ptr, np.int32), t(cov, np.int32)
            outs = {name: (torch.zeros(nq * ncov, dtype=torch.float64, device=dev), torch.zeros(nq, dtype=torch.float32, device=dev))
                    for name in libs}
            torch.cuda.synchronize()

            def run(name, k):
                for _ in range(k):
                    rc = libs[name].orbfe_bow_min_score_device(vocs[name], nq, F, cap, d_ids.data_ptr(), d_vals.data_ptr(), d_n.data_ptr(),
                                                               d_q.data_ptr(), d_ptr.data_ptr(), d_cov.data_ptr(), outs[name][0].data_ptr(),
                                                               outs[name][1].data_ptr(), stream.cuda_stream)
                    assert rc == 0
            times = {name: [] for name in libs}
            for name in libs:
                run(name, 10 * args.warmup)
            stream.synchronize()
            for _ in range(5):                       # alternate the builds
                for name in libs:
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(stream)
                    run(name, reps)
                    e1.record(stream)
                    stream.synchronize()
                    times[name].append(e0.elapsed_time(e1) / reps * 1e3)
            key = "%dq_x_%dcov" % (nq, ncov)
            for name in libs:
                res["%s_%s_us" % (key, name)] = [round(min(times[name]), 2), round(max(times[name]), 2)]   # least and most of 5 rounds
            if "baseline" in libs:
                res[key + "_same_bits"] = bool(torch.equal(outs["this"][0].view(torch.int64), outs["baseline"][0].view(torch.int64)) and
                                               torch.equal(outs["this"][1].view(torch.int32), outs["baseline"][1].view(torch.int32)))
            if nq == 1:
                d_rows = t(np.concatenate([qrow, cov]), np.int64)

                def host_path():
                    hi, hv, hn = d_ids[d_rows].cpu().numpy(), d_vals[d_rows].cpu().numpy(), d_n[d_rows].cpu().numpy()
                    m = np.float32(1)
                    for k in range(1, len(hn)):
                        sc = np.float32(OS.bow_score(hi[0, :hn[0]], hv[0, :hn[0]], hi[k, :hn[k]], hv[k, :hn[k]]))
                        if sc < m:
                            m = sc
                    d_m = torch.tensor([m], dtype=torch.float32).to(dev, non_blocking=True)
                    torch.cuda.synchronize()
                    return m, d_m
                m, _ = host_path()
                t0 = time.perf_counter()
                for _ in range(5 * args.iters):
                    host_path()
                res[key + "_host_path_us"] = round((time.perf_counter() - t0) / (5 * args.iters) * 1e6, 1)
                res[key + "_host_same_min"] = bool(np.float32(m).tobytes() == outs["this"][1].cpu().numpy()[0].tobytes())
        out["%d_words" % wpk] = res
    for name, L in libs.items():
        L.orbfe_vocabulary_destroy(vocs[name])
    return out


def vocload(args):
    import tempfile
    import torch
    from torch.profiler import profile, ProfilerActivity
    from orb_slam_b200 import bow as BW
    from orb_slam_b200.synth import random_vocabulary
    from oracle import voc_text as VT
    torch.zeros(1, device="cuda")
    voc = random_vocabulary(10, 6, seed=3)
    nd, cp, ch = voc["node_desc"], voc["child_ptr"], voc["children"]
    n = len(nd)
    parent = np.zeros(n, np.int64)
    parent[ch] = np.repeat(np.arange(n), np.diff(cp))
    leaf = (np.diff(cp) == 0).astype(int)
    desc = [" ".join(map(str, row)) for row in nd.tolist()]
    w = voc["weight"].tolist()
    out = {"what": "orbfe_vocabulary_load_text, k=10 L=6 synthetic text (%d nodes), %d iterations after %d warm-up" % (n, args.iters, args.warmup)}
    with tempfile.TemporaryDirectory() as tmp:
        for name, fmt in (("orbvoc_like", lambda i: "%.6g" % w[i] if leaf[i] else "0"), ("repr_weights", lambda i: repr(w[i]))):
            path = os.path.join(tmp, name + ".txt")
            with open(path, "w") as f:
                f.write("10 6 0 0\n" + "".join("%d %d %s  %s\n" % (parent[i], leaf[i], desc[i], fmt(i)) for i in range(1, n)))
            res = {"bytes": os.path.getsize(path)}
            for _ in range(args.warmup):
                BW.Vocabulary.load_text(path).close()
            walls = []
            for _ in range(args.iters):
                t0 = time.perf_counter()
                V = BW.Vocabulary.load_text(path)
                walls.append(time.perf_counter() - t0)
                V.close()
            res["load_text_wall_ms"] = {"min": round(1e3 * min(walls), 2), "median": round(1e3 * float(np.median(walls)), 2),
                                        "max": round(1e3 * max(walls), 2)}
            t0 = time.perf_counter()
            open(path, "rb").read()
            res["file_read_only_ms"] = round(1e3 * (time.perf_counter() - t0), 2)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                BW.Vocabulary.load_text(path).close()
            dev = {}
            for e in prof.key_averages():
                t = getattr(e, "device_time_total", 0)
                if t > 0:
                    dev[e.key.replace("orbfe::(anonymous namespace)::", "").split("(")[0].strip()[:60]] = {"calls": e.count, "us": round(t, 1)}
            res["device_us"] = dev
            ref_path = VT.text_for_reference(path, os.path.join(tmp, "ref.txt"))
            ref = VT.RefVocabularyNodes(ref_path)
            res["reference_loadFromTextFile_ms"] = round(1e3 * ref.seconds, 1)
            ref.close()
            os.remove(ref_path)
            out[name] = res
    _gpu_and_power_limit(out)
    return out


def normaldepth(args):
    """MapPoint::UpdateNormalAndDepth at the end of LocalBundleAdjustment (Optimizer.cc:488): after the optimisation every
    local map point gets SetWorldPos and then UpdateNormalAndDepth.  The local map: 20 keyframes of 2000 features whose every
    feature is a map point, 10000 points, each observed by 2-60 keyframes of a 60-keyframe store (95 % in 2-12, in keyframe
    order), world positions 2-40 units in front of their reference keyframe.  CUDA-event ms of orbfe_normal_and_depth_device
    on the frame store, the wall time of orbfe_normal_and_depth including the host gather of every observer's centre, and
    the wall time of the oracle's C loop (oracle/orb_oracle_normal_depth.c: plain C, not OpenCV) on the same host arrays."""
    import torch
    import orb_slam_b200 as fe
    from orb_slam_b200 import bow as BW
    from oracle import normal_depth as ND
    NKF, NF, NP = 60, 2000, 10000
    rng = np.random.default_rng(17)
    counts = np.full(NKF, NF, np.int32)
    octs = rng.integers(0, 8, NKF * NF).astype(np.int32)
    kps = np.zeros(NKF * NF, fe.KP_DTYPE)
    kps["octave"] = octs
    centers = (rng.standard_normal((NKF, 3)) * 3).astype(np.float32)
    n_obs = np.where(rng.random(NP) < 0.95, rng.integers(2, 13, NP), rng.integers(13, 61, NP))
    groups, ref = [], np.zeros(NP, np.int32)
    for p in range(NP):
        frames = np.sort(rng.choice(NKF, int(n_obs[p]), replace=False))
        g = frames * NF + rng.integers(0, NF, len(frames))
        groups.append(g.astype(np.int32))
        ref[p] = g[rng.integers(0, len(g))]
    gp = np.concatenate([[0], np.cumsum([len(g) for g in groups])]).astype(np.int32)
    obs = np.concatenate(groups).astype(np.int32)
    d = rng.standard_normal((NP, 3))
    world = (centers[ref // NF] + d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(2, 40, (NP, 1))).astype(np.float32)
    t = [np.float32(1.0)]                      # Frame.cc:90-103: the float chain of the extractor's scale factor
    for _ in range(7):
        t.append(np.float32(t[-1] * np.float32(1.2)))
    sfs = np.array(t, np.float32)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    s = stream.cuda_stream
    tt = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d_kps, d_cnt, d_c, d_gp, d_obs, d_ref, d_w = tt(kps.view(np.uint8)), tt(counts), tt(centers), tt(gp), tt(obs), tt(ref), tt(world)
    d_n = torch.zeros((NP, 3), dtype=torch.float32, device=dev)
    d_a, d_b = torch.zeros(NP, dtype=torch.float32, device=dev), torch.zeros(NP, dtype=torch.float32, device=dev)
    m = fe.ORBmatcher(0.6, True)
    call = lambda: BW.normal_and_depth_device(m, NP, d_kps.data_ptr(), d_cnt.data_ptr(), NKF, NF, d_c.data_ptr(), d_gp.data_ptr(),
                                              d_obs.data_ptr(), len(obs), d_w.data_ptr(), d_ref.data_ptr(), 1.2, sfs, d_n.data_ptr(),
                                              d_a.data_ptr(), d_b.data_ptr(), s)
    out = {"what": "UpdateNormalAndDepth after a local BA: %d map points, %d observations (max %d per point) over a %d-keyframe store "
                   "of %d features" % (NP, len(obs), int(n_obs.max()), NKF, NF)}
    for _ in range(max(args.warmup, 3)):
        call()
    stream.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    iters = args.iters * 20
    times = []
    for _ in range(5):
        e0.record(stream)
        for _ in range(iters):
            call()
        e1.record(stream)
        stream.synchronize()
        times.append(e0.elapsed_time(e1) / iters)
    m.sync()
    out["device_ms"] = float(np.median(times))
    out["device_ms_min_max"] = [float(min(times)), float(max(times))]
    got = (d_n.cpu().numpy(), d_a.cpu().numpy(), d_b.cpu().numpy())
    lat, host, orc = [], None, []
    for _ in range(7):
        t0 = time.perf_counter()
        host = BW.normal_and_depth(m, world, centers[ref // NF], octs[ref], gp, centers[obs // NF], 1.2, sfs)
        lat.append((time.perf_counter() - t0) * 1e3)
    out["host_entry_with_gather_wall_ms"] = float(np.median(lat))
    want = None
    rc, ro, oc = centers[ref // NF], octs[ref], centers[obs // NF]
    for _ in range(3):
        t0 = time.perf_counter()
        want = ND.normal_depth(world, rc, ro, gp, oc, 1.2, sfs)
        orc.append((time.perf_counter() - t0) * 1e3)
    out["oracle_c_loop_wall_ms_not_opencv"] = float(np.median(orc))
    same = lambda x, y: all(np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(np.nan_to_num(a), np.nan_to_num(b))
                            for a, b in zip(x, y))
    out["same_as_host"] = bool(same(got, host))
    out["same_as_oracle"] = bool(same(got, want))
    _gpu_and_power_limit(out)
    m.close()
    return out


def covis(args):
    """UpdateConnections of one keyframe and of 64 keyframes of a 2000-keyframe map, each keyframe already updated once (a
    repeated call leaves the graph as it is, so every timed call does the same work)."""
    import torch
    from orb_slam_b200 import bow as BW
    from oracle.covis import CovisOracle
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
    import covis_scenes as CS
    scene = CS.scene_large()
    K, cap = scene.nkf, scene.cap
    slot_of = scene.slots()
    model = CS.Model(scene)
    for st in scene.steps:
        model.apply(st)
    kf_mp, counts, gp, obs = model.inputs(slot_of, K)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    s = stream.cuda_stream
    tt = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d_mp, d_cnt, d_gp, d_obs = tt(kf_mp), tt(counts), tt(gp), tt(obs)
    g = BW.CovisibilityGraph(K, 64, 64)
    orc = CovisOracle(K)
    g.add(slot_of, np.arange(K), np.arange(K))
    for k in range(K):
        orc.add(slot_of[k], k, k)
    upd = lambda sl: g.update_connections_device(sl, d_mp.data_ptr(), d_cnt.data_ptr(), K, cap, d_gp.data_ptr(), d_obs.data_ptr(),
                                                 len(gp) - 1, len(obs), stream=s)
    order = [int(slot_of[k]) for k in range(K)]
    for b in range(0, K, 64):
        upd(order[b:b + 64])
    orc.replay(order, kf_mp, counts, cap, gp, obs)
    g.sync()
    out = {"what": "UpdateConnections on a %d-keyframe map of %d features, %d points, %d observations" % (K, cap, len(gp) - 1, len(obs))}
    mid = K // 2
    for name, sl in (("batch1", order[mid:mid + 1]), ("batch64", order[mid:mid + 64])):
        for _ in range(max(args.warmup, 3)):
            upd(sl)
        stream.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        iters = args.iters * 20
        times = []
        for _ in range(5):
            e0.record(stream)
            for _ in range(iters):
                upd(sl)
            e1.record(stream)
            stream.synchronize()
            times.append(e0.elapsed_time(e1) / iters)
        g.sync()
        out[name + "_device_ms"] = float(np.median(times))
        out[name + "_device_ms_min_max"] = [float(min(times)), float(max(times))]
        orc_ms = []
        for _ in range(3):
            t0 = time.perf_counter()
            orc.replay(sl, kf_mp, counts, cap, gp, obs)
            orc_ms.append((time.perf_counter() - t0) * 1e3)
        out[name + "_oracle_c_wall_ms_not_reference"] = float(np.median(orc_ms))
    g.close()
    orc.close()
    _gpu_and_power_limit(out)
    return out


def observations(args):
    """the lists of the points of one keyframe and of every point of a 2000-keyframe map, on the device and on the host
    from the reference's own maps"""
    import torch
    from orb_slam_b200 import bow as BW
    from oracle import observations as OO
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
    import covis_scenes as CS
    scene = CS.scene_large()
    K, cap = scene.nkf, scene.cap
    slot_of = scene.slots()
    model = CS.Model(scene)
    ref = OO.RefObservations()
    for st in scene.steps:
        model.apply(st)
        if st[0] == "kf":
            ref.add_keyframe(st[1])
        elif st[0] == "pts":
            ref.add_points(st[1])
            ref.observe_many(st[2], st[3], st[4])
    kf_mp, counts, gp, obs = model.inputs(slot_of, K)
    npts = len(gp) - 1
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    tt = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d_mp, d_cnt = tt(kf_mp), tt(counts)
    g = BW.CovisibilityGraph(K, 64, 64)
    g.add(slot_of, np.arange(K), np.arange(K))
    row = kf_mp[int(slot_of[K // 2]) * cap:(int(slot_of[K // 2]) + 1) * cap]
    out = {"what": "GetObservations lists on a %d-keyframe map of %d features, %d points, %d observations" % (K, cap, npts, len(obs))}
    for name, pts in (("one_keyframe", np.unique(row[row >= 0]).astype(np.int32)), ("all_points", np.arange(npts, dtype=np.int32))):
        n = len(pts)
        d_pts, d_rs = tt(pts), tt(np.zeros(n, np.int32))
        z = lambda k: torch.zeros(max(k, 1), dtype=torch.int32, device=dev)
        d_ptr, d_obs, d_nobs, d_ro = z(n + 1), z(len(obs)), z(1), z(n)
        d_scr = torch.zeros(BW.CovisibilityGraph.observations_scratch_bytes(npts, K, cap, len(obs)) // 4 + 1, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        call = lambda: g.observations_device(n, d_pts.data_ptr(), npts, d_mp.data_ptr(), d_cnt.data_ptr(), K, cap, len(obs), d_ptr.data_ptr(),
                                             d_obs.data_ptr(), d_nobs.data_ptr(), d_scr.data_ptr(), d_rs.data_ptr(), d_ro.data_ptr(),
                                             stream.cuda_stream)
        for _ in range(max(args.warmup, 3)):
            call()
        stream.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        iters = args.iters * 20
        times = []
        for _ in range(5):
            e0.record(stream)
            for _ in range(iters):
                call()
            e1.record(stream)
            stream.synchronize()
            times.append(e0.elapsed_time(e1) / iters)
        g.sync()
        out[name + "_points"] = n
        out[name + "_device_ms"] = float(np.median(times))
        out[name + "_device_ms_min_max"] = [float(min(times)), float(max(times))]
        hptr, hobs = np.zeros(n + 1, np.int32), np.zeros(max(len(obs), 1), np.int32)
        host_ms = []
        for _ in range(3):
            t0 = time.perf_counter()
            tot = ref.flatten(pts, slot_of, cap, hptr, hobs)
            host_ms.append((time.perf_counter() - t0) * 1e3)
        out[name + "_host_from_reference_maps_wall_ms"] = float(np.median(host_ms))
        nd = int(d_nobs.item())
        out[name + "_lists_equal"] = bool(nd == tot and np.array_equal(d_ptr.cpu().numpy(), hptr) and
                                          np.array_equal(d_obs.cpu().numpy()[:nd], hobs[:tot]))
    g.close()
    ref.close()
    _gpu_and_power_limit(out)
    return out


def kfculling(args):
    """one KeyFrameCulling call on the device, the oracle and the reference, for three list lengths and three cull places"""
    import torch
    from orb_slam_b200 import bow as BW
    from oracle import kf_culling as KC
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
    import covis_scenes as CS
    import kf_culling_scenes as KS
    from test_oracle_kf_culling import cull_inputs
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    tt = lambda a, dt=np.int32: torch.from_numpy(np.ascontiguousarray(a, dt)).to(dev)
    C = 256
    out = {"what": "KeyFrameCulling for one current keyframe of a 2000-keyframe x 2000-feature map; ms per call"}
    for window in (5, 25, 64):
        scene = CS.scene_large(window=window)
        K, cap = scene.nkf, scene.cap
        slot_of = scene.slots()
        model = KS.CullModel(scene)
        g = BW.CovisibilityGraph(K, C, 64)
        g.add(slot_of, np.arange(K), np.arange(K))
        ref = KC.RefKfCulling() if KC.ref_available() else None
        for st in scene.steps:
            model.apply(st)
            if st[0] == "update":
                kf_mp, counts, gp, obs = model.inputs(slot_of, K)
                d = [tt(kf_mp), tt(counts), tt(gp), tt(obs)]
                g.update_connections_device([int(slot_of[k]) for k in st[1]], d[0].data_ptr(), d[1].data_ptr(), K, cap, d[2].data_ptr(),
                                            d[3].data_ptr(), len(gp) - 1, len(obs))
            if ref is not None:
                if st[0] == "kf":
                    ref.add_keyframe(st[1])
                elif st[0] == "pts":
                    ref.add_points(st[1])
                    ref.observe_many(st[2], st[3], st[4])
                elif st[0] == "update":
                    for k in st[1]:
                        ref.update(k)
        g.sync()
        cur = K // 2
        a = cull_inputs(model, slot_of, K)
        npts = len(a["point_bad"])
        d_lp, d_l = torch.zeros(2, dtype=torch.int32, device=dev), torch.zeros(C, dtype=torch.int32, device=dev)
        g.lists_device(0, [int(slot_of[cur])], 0, d_lp.data_ptr(), d_l.data_ptr())
        g.sync()
        n = int(d_lp[1].item())
        lst = d_l.cpu().numpy()[:n]
        kf_of = np.argsort(slot_of)
        obs_cap = int(np.count_nonzero(a["kf_mp"] >= 0))
        pristine = dict(kf_mp=tt(a["kf_mp"]), point_bad=tt(a["point_bad"], np.uint8), ref_slot=tt(a["ref_slot"]))
        work = {k: v.clone() for k, v in pristine.items()}
        kp = np.zeros(K * cap, dtype=__import__("orb_slam_b200").KP_DTYPE)
        kp["octave"] = a["octave"]
        d_cnt, d_kps = tt(a["counts"]), tt(kp.view(np.uint8), np.uint8)
        z = lambda k: torch.zeros(max(k, 1), dtype=torch.int32, device=dev)
        o_nobs, o_vs, o_vd, o_nc, o_bp, o_nb = z(1), z(C), z(C), z(1), z(npts), z(1)
        d_scr = z(BW.CovisibilityGraph.cull_scratch_bytes(npts, K, cap, obs_cap) // 4 + 1)
        tag = "covisibles_%d" % n
        for place, allowed in (("front", lst[:5]), ("middle", lst[n // 2:n // 2 + 5]), ("nowhere", lst[:0])):
            ne = [int(s) for s in lst if s not in set(allowed.tolist())]
            times = []
            for it in range(max(args.warmup, 2) + 5):
                for k in work:
                    work[k].copy_(pristine[k])
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record(stream)
                g.keyframe_culling_device(int(slot_of[cur]), work["kf_mp"].data_ptr(), d_cnt.data_ptr(), d_kps.data_ptr(), K, cap,
                                          work["point_bad"].data_ptr(), work["ref_slot"].data_ptr(), npts, ne, obs_cap, o_nobs.data_ptr(),
                                          o_vs.data_ptr(), o_vd.data_ptr(), o_nc.data_ptr(), o_bp.data_ptr(), o_nb.data_ptr(), d_scr.data_ptr(),
                                          stream=stream.cuda_stream)
                e1.record(stream)
                stream.synchronize()
                if it >= max(args.warmup, 2):
                    times.append(e0.elapsed_time(e1))
            g.sync()
            ne_flags = a["not_erase"].copy()
            ne_flags[ne] = 1
            t0 = time.perf_counter()
            o = KC.cull(lst, a["live"], a["id0"], a["keys"], ne_flags, a["kf_mp"], a["counts"], a["octave"], cap, a["point_bad"],
                        a["ref_slot"])
            out[tag + "_" + place + "_oracle_wall_ms"] = (time.perf_counter() - t0) * 1e3
            out[tag + "_" + place + "_device_ms"] = float(np.median(times))
            out[tag + "_" + place + "_device_ms_min_max"] = [float(min(times)), float(max(times))]
            vd = o_vd.cpu().numpy()[:n]
            out[tag + "_" + place + "_erased"] = int((vd == KC.ERASED).sum())
            out[tag + "_" + place + "_made_bad"] = int(o_nb.item())
            out[tag + "_" + place + "_equals_oracle"] = bool(o["status"] == 0 and vd.tolist() == o["verdict"].tolist() and
                                                             np.array_equal(work["kf_mp"].cpu().numpy(), o["kf_mp"]))
            if place == "nowhere" and ref is not None:
                for s in ne:
                    ref.set_not_erase(int(kf_of[s]))
                ids, verdicts, ns = ref.cull(cur)
                out[tag + "_nowhere_reference_wall_ms"] = ns / 1e6
                out[tag + "_nowhere_reference_verdicts_equal"] = verdicts == vd.tolist() and [int(slot_of[i]) for i in ids] == lst.tolist()
        g.close()
        if ref is not None:
            ref.close()
    _gpu_and_power_limit(out)
    return out


def localmap(args):
    """one UpdateReference call on the device and in the reference, for three frame sizes"""
    import torch
    from orb_slam_b200 import bow as BW
    from oracle import local_map as LM
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
    import covis_scenes as CS
    import local_map_scenes as LS
    from test_oracle_local_map import lm_inputs
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    tt = lambda a, dt=np.int32: torch.from_numpy(np.ascontiguousarray(a, dt)).to(dev)
    scene = CS.scene_large()
    K, cap = scene.nkf, scene.cap
    slot_of = scene.slots()
    model = LS.LmModel(scene)
    g = BW.CovisibilityGraph(K, 64, 64)
    g.add(slot_of, np.arange(K), np.arange(K))
    ref = LM.RefLocalMap() if LM.ref_available() else None
    for st in scene.steps:
        model.apply(st)
        if st[0] == "update":
            kf_mp, counts, gp, obs = model.inputs(slot_of, K)
            d = [tt(kf_mp), tt(counts), tt(gp), tt(obs)]
            g.update_connections_device([int(slot_of[k]) for k in st[1]], d[0].data_ptr(), d[1].data_ptr(), K, cap, d[2].data_ptr(),
                                        d[3].data_ptr(), len(gp) - 1, len(obs))
        if ref is not None:
            if st[0] == "kf":
                ref.add_keyframe(st[1])
            elif st[0] == "pts":
                ref.add_points(st[1])
                ref.observe_many(st[2], st[3], st[4])
            elif st[0] == "update":
                for k in st[1]:
                    ref.update(k)
    g.sync()
    a = lm_inputs(model, slot_of, K)
    npts = len(a["point_bad"])
    d_kf_mp, d_cnt, d_pb = tt(a["kf_mp"]), tt(a["counts"]), tt(a["point_bad"], np.uint8)
    z = lambda k: torch.zeros(max(k, 1), dtype=torch.int32, device=dev)
    d_lk, d_nlk, d_ref, d_lp, d_nlp = z(K), z(1), z(1), z(npts), z(1)
    d_scr = z(BW.CovisibilityGraph.local_map_scratch_bytes(npts, K) // 4 + 1)
    out = {"what": "Tracking::UpdateReference for one frame on a %d-keyframe x %d-feature map (%d points); ms per call" % (K, cap, npts)}
    for cells in LS.large_frames(model, slot_of):
        tag = "frame_%d" % len(cells)
        d_frame = tt(cells)
        times = []
        for it in range(max(args.warmup, 2) + 20):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record(stream)
            g.local_map_device(len(cells), d_frame.data_ptr(), d_pb.data_ptr(), npts, d_kf_mp.data_ptr(), d_cnt.data_ptr(), K, cap,
                               d_lk.data_ptr(), d_nlk.data_ptr(), d_ref.data_ptr(), d_lp.data_ptr(), d_nlp.data_ptr(), d_scr.data_ptr(),
                               stream=stream.cuda_stream)
            e1.record(stream)
            stream.synchronize()
            if it >= max(args.warmup, 2):
                times.append(e0.elapsed_time(e1))
        g.sync()
        nlk, nlp = int(d_nlk.item()), int(d_nlp.item())
        out[tag + "_device_ms"] = float(np.median(times))
        out[tag + "_device_ms_min_max"] = [float(min(times)), float(max(times))]
        out[tag + "_local_keyframes"] = nlk
        out[tag + "_local_points"] = nlp
        if ref is not None:
            fm, lk, rk, lp, ns = ref.update_reference(cells)
            out[tag + "_reference_wall_ms"] = ns / 1e6
            out[tag + "_equals_reference"] = bool(d_lk.cpu().numpy()[:nlk].tolist() == [int(slot_of[k]) for k in lk] and
                                                  d_lp.cpu().numpy()[:nlp].tolist() == lp and int(d_ref.item()) == int(slot_of[rk]))
        else:
            out[tag + "_reference_wall_ms"] = "not measured: oracle/_ref/libref_local_map.so absent"
    g.close()
    if ref is not None:
        ref.close()
    _gpu_and_power_limit(out)
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--what", default="config3,config5")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--groups", type=int, default=10000)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--baseline-lib", default=None, help="--what guided, kfdbbatch, loopscore: another build of liborbfe.so to time alternately")
    args = ap.parse_args()
    for w in args.what.split(","):
        print(json.dumps({"config3": config3, "config5": config5, "small": small, "exchange1": exchange1, "matchers": matchers, "h2d": h2d, "fast": fast, "latency": latency,
                          "reloc": reloc, "mapping": mapping, "mapdesc": mapdesc, "kfdb": kfdb, "kfdbbatch": kfdbbatch, "bowchain": bowchain,
                          "windowed": windowed, "guided": guided, "loopscore": loopscore, "vocload": vocload,
                          "normaldepth": normaldepth, "covis": covis, "observations": observations, "kfculling": kfculling,
                          "localmap": localmap, "multigeom": multigeom, "multitrack": multitrack}[w](args)))
