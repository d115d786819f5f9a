"""What skipping the loop filter (include/edge264_loopfilter.h, edge264_set_loop_filter) saves on the GPU, on bench.py's
1080p workload (its streams and seeds), in the modes ALL (the default), REF (non-reference pictures unfiltered) and NONE.

1. Kernel-only replay: the streams decoded once as bench.py does (tools/libe264bench.so, records kept with E264B_KEEP=1),
   once per mode (E264_BENCH_LOOP_FILTER=<mode>); then e264b_replay of each set of decoders, modes alternating,
   `--runs` times each, as tools/replay_ab.py does.  Frames per second of device time, and the mean span per launch of
   each kernel kind.
2. torch.profiler with CUDA activities over a few streams per mode, in a pass of its own: device time per picture of
   every kernel and copy.
3. Host-to-device and device-to-host bytes and kernel launches per picture (e264b_stats) of the decodes of step 1.
4. End to end: the same streams with the README loop, one decoder per stream (n_threads 0), one Python thread per CPU,
   modes alternating, `--runs` times each.  Host CABAC parsing bounds this figure, so no gain is expected here.
5. The card's name and power limit, read in the same run.

It needs a CUDA device and fails without one.  It reads `nvidia-smi --query-gpu` and changes no device setting.

  python tools/loop_filter_cost.py --out results/h100_loop_filter_cost_1080p.txt
"""
import argparse, ctypes, errno, os, queue, subprocess, sys, tempfile, threading, time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import edge264_b200 as pkg  # noqa: E402

MODES = [("all", pkg.LOOP_FILTER_ALL), ("ref", pkg.LOOP_FILTER_REF), ("none", pkg.LOOP_FILTER_NONE)]


def decode_one(lib, data, mode):
    buf = ctypes.create_string_buffer(data, len(data) + 64)
    base = ctypes.addressof(buf); end = base + len(data)
    dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
    if not dec:
        raise RuntimeError("edge264_alloc failed (no CUDA device: the GPU backend has no CPU fallback)")
    if lib.edge264_set_loop_filter(dec, mode):
        raise RuntimeError("edge264_set_loop_filter failed")
    nal, n, f = base + 3 + (1 if data[2] == 0 else 0), 0, pkg.Edge264Frame()
    while True:
        sc = lib.edge264_find_start_code(nal, end, 0) if nal < end else end
        res = lib.edge264_decode_NAL(dec, nal, sc, None, None)
        while lib.edge264_get_frame(dec, ctypes.byref(f), 0) == 0:
            n += 1
        if res == errno.ENOBUFS:
            continue
        if nal >= end:
            break
        nal = sc + 3 if sc + 3 < end else end
    d = ctypes.c_void_p(dec)
    lib.edge264_free(ctypes.byref(d))
    return n


def e2e(lib, bufs, mode, threads):
    q = queue.Queue()
    for b in bufs:
        q.put(b)
    counts = []
    def work():
        while True:
            try:
                b = q.get_nowait()
            except queue.Empty:
                return
            counts.append(decode_one(lib, b, mode))
    t0 = time.perf_counter()
    th = [threading.Thread(target=work) for _ in range(threads)]
    for t in th: t.start()
    for t in th: t.join()
    return sum(counts), time.perf_counter() - t0


def profile(lib, bufs, mode):
    import torch
    from torch.profiler import profile as tprof, ProfilerActivity
    with tprof(activities=[ProfilerActivity.CUDA]) as p:
        frames = sum(decode_one(lib, b, mode) for b in bufs)
        torch.cuda.synchronize()
    per = {}
    for e in p.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:   # kernels, copies and memsets, with their device time
            name = e.name.split("(")[0]
            per.setdefault(name[5:] if name.startswith("void ") else name, []).append(e.time_range.elapsed_us())
    return frames, per


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=32); ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--replay-streams", type=int, default=16); ap.add_argument("--replay-steps", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3); ap.add_argument("--threads", type=int, default=len(os.sched_getaffinity(0)))
    ap.add_argument("--profile-streams", type=int, default=2); ap.add_argument("--out", required=True)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("loop_filter_cost.py measures on a CUDA device; none is available")
    torch.cuda.init()
    lines = []
    def say(s):
        print(s, flush=True); lines.append(s)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    say("card: %s (name, power limit; read in this run)" % card.splitlines()[0] if card else "card: nvidia-smi gave nothing")
    cfg = bench.CONFIGS["1080p"]
    bufs = bench.generate_streams(cfg, [cfg["seed0"] + i for i in range(a.streams)], a.frames, tempfile.mkdtemp(prefix="e264_loop_filter_cost"))
    say("workload: bench.py 1080p, %d streams x %d frames, %dx%d (%s)" % (len(bufs), a.frames, cfg["w"] * 16, cfg["h"] * 16, cfg["gen"]))
    lib = pkg.load()
    core = ctypes.CDLL(pkg.LIB_PATH)
    core.e264b_of_decoder.restype = ctypes.c_void_p; core.e264b_of_decoder.argtypes = [ctypes.c_void_p]
    core.e264b_replay.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.POINTER(bench.ReplayStats)]
    core.e264b_stats.argtypes = [ctypes.c_void_p] + [ctypes.POINTER(ctypes.c_uint64)] * 3
    core.e264b_error_flag.argtypes = [ctypes.c_void_p]
    blib = bench.BenchLib(os.path.join(ROOT, "tools", "libe264bench.so"))

    # ---- 1 and 3: decoders kept by the benchmark's loop, their counts, then the kernel-only replay ----
    S = min(a.replay_streams, len(bufs))
    os.environ["E264B_KEEP"] = "1"
    kept = {}
    for m, mode in MODES:
        os.environ["E264_BENCH_LOOP_FILTER"] = str(mode)
        secs, frames, sums, decs = blib.run(bufs[:S], min(S, 16), keep=True)
        devs = (ctypes.c_void_p * S)(*[core.e264b_of_decoder(decs[i]) for i in range(S)])
        tot = [0, 0, 0]
        for i in range(S):
            v = [ctypes.c_uint64() for _ in range(3)]
            core.e264b_stats(devs[i], *[ctypes.byref(x) for x in v])
            tot = [t + x.value for t, x in zip(tot, v)]
        n = sum(frames)
        say("counts %-10s %d pictures: kernel launches %.2f, host-to-device %.0f bytes, device-to-host %.0f bytes per picture" % (m, n, tot[0] / n, tot[1] / n, tot[2] / n))
        kept[m] = (decs, devs, n)
    os.environ.pop("E264_BENCH_LOOP_FILTER", None); os.environ["E264B_KEEP"] = "0"
    T = 8
    for m, _ in MODES:     # warm-up: graph capture, module loads
        st = bench.ReplayStats()
        if core.e264b_replay(kept[m][1], S, 1, T, ctypes.byref(st)):
            raise SystemExit("e264b_replay failed")
    rep = {m: [] for m, _ in MODES}
    for r in range(a.runs):
        for m, _ in MODES:
            decs, devs, n = kept[m]
            st = bench.ReplayStats()
            if core.e264b_replay(devs, S, a.replay_steps, T, ctypes.byref(st)) or any(core.e264b_error_flag(devs[i]) for i in range(S)):
                raise SystemExit("e264b_replay failed")
            fps = n * a.replay_steps / st.ms_total * 1000
            rep[m].append(fps)
            per = " ".join("%s %.0f us" % (k, 1000 * st.kernel_ms[i] / max(1, st.kernel_launches[i])) for i, k in ((1, "inter"), (2, "intra"), (3, "deblock")))
            say("replay run %d %-10s %d streams in flight: %.1f ms per step, %.0f frames/s; mean span per launch: %s" % (r + 1, m, S, st.ms_total / a.replay_steps, fps, per))
    for m, _ in MODES:
        v = sorted(rep[m])
        say("replay %-10s median %.0f frames/s (min %.0f, max %.0f)" % (m, v[len(v) // 2], v[0], v[-1]))
    for m, _ in MODES:
        blib.free(kept[m][0])

    # ---- 2: device time per picture per kernel ----
    for m, mode in MODES:
        frames, per = profile(lib, bufs[:a.profile_streams], mode)
        say("torch.profiler, %d streams, %s (%d pictures): device time, us" % (a.profile_streams, m, frames))
        tot = 0.0
        for k in sorted(per):
            v = per[k]
            tot += sum(v)
            say("  %-60s launches %5d  mean %8.2f  total per picture %8.2f" % (k, len(v), sum(v) / len(v), sum(v) / frames))
        say("  %-60s %8.2f" % ("all of the above, per picture", tot / frames))

    # ---- 4: end to end ----
    say("end to end: %d streams, %d host threads, one decoder per stream (n_threads 0)" % (len(bufs), a.threads))
    for _, mode in MODES:       # warm-up: device contexts, pinned buffers, code pages
        e2e(lib, bufs[:a.threads], mode, a.threads)
    res = {m: [] for m, _ in MODES}
    for r in range(a.runs):
        for m, mode in MODES:
            n, dt = e2e(lib, bufs, mode, a.threads)
            res[m].append(n / dt)
            say("e2e run %d %-10s %d frames in %.3f s  %.1f frames/s" % (r + 1, m, n, dt, n / dt))
    for m, _ in MODES:
        v = sorted(res[m])
        say("e2e %-10s median %.1f frames/s (min %.1f, max %.1f)" % (m, v[len(v) // 2], v[0], v[-1]))
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fo:
        fo.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
