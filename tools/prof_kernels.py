#!/usr/bin/env python3
"""Measurement harness for the configurations that are not the bench line (run on one H100):

  --what config3   BASELINE configs[2]: 3840x2160, 4000 kp, 12 levels -- per-stage CUDA-event times of the extractor on a
                   device-resident batch, achieved GB/s against the 130.86 MB/frame of SURVEY.md 8(d)
  --what config5   BASELINE configs[4]: 2000 query descriptors x (ngroups keyframes x 2000 descriptors): the brute-force
                   best/second sweep (knn2 kernel), Gpairs/s, HBM GB/s, POPC-pipe estimate
  --what small     the latency-bound kernels once each (bow_descend, distinctive, undistort, hamming_csr, sbp single pair)
                   so that an `ncu -k regex:` capture finds them

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
        V.close()
    except Exception as e:
        out["bow"] = "skipped: %r" % e
    ex.close(); m.close()
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


def fastarc(args):
    """BASELINE configs[1] geometry (1920x1080, 2000 kp, 8 levels), 64-frame device-resident batches: per-stage CUDA-event
    times for every compiled FAST arc-network variant (ORBFE_FAST_ARC is read when the extractor plans a geometry)."""
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
    out = {"what": "FAST arc-network variants, 1080p x 64 frames, ms per batch"}
    ref = None
    # "arc" or "arc:ctas" (ctas = resident CTAs per SM, 4 x 64 registers or 3 x 80)
    variants = [v for v in os.environ.get("FASTARC_VARIANTS", "-1,0,4,8,12,16,12:3,16:3").split(",")]
    for rep in range(2):
        for var in variants:
            arc, _, ctas = var.partition(":")
            arc = int(arc)
            os.environ["ORBFE_FAST_ARC"] = str(arc)
            if ctas:
                os.environ["ORBFE_FAST_CTAS"] = ctas
            else:
                os.environ.pop("ORBFE_FAST_CTAS", None)
            ex = fe.ORBextractor(NF, 1.2, NL, fe.FAST_SCORE, 20)
            ex.set_profiling(True)
            for _ in range(3):
                ex.extract_batch_device(d_frames.data_ptr(), W, H, W, W * H, B, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), stream.cuda_stream)
            stream.synchronize()
            ex.stage_times()
            n = 10
            for _ in range(n):
                ex.extract_batch_device(d_frames.data_ptr(), W, H, W, W * H, B, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr(), stream.cuda_stream)
            stream.synchronize()
            acc = {}
            for name, ms in ex.stage_times():
                acc[name] = acc.get(name, 0.0) + ms / n
            sig = (d_kps.cpu().numpy().tobytes(), d_desc.cpu().numpy().tobytes())
            if ref is None:
                ref = sig
            out["arc%s_rep%d" % (var, rep)] = {"fast_nms": round(acc.get("fast_nms", -1), 4), "all": round(sum(acc.values()), 4), "same_bits": sig == ref}
            ex.close()
    os.environ.pop("ORBFE_FAST_ARC", None)
    os.environ.pop("ORBFE_FAST_CTAS", None)
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


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--what", default="config3,config5")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--groups", type=int, default=10000)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    for w in args.what.split(","):
        print(json.dumps({"config3": config3, "config5": config5, "small": small, "exchange1": exchange1, "matchers": matchers, "h2d": h2d, "fastarc": fastarc, "latency": latency}[w](args)))
