"""What skipping pictures (include/edge264_skip.h) saves, on bench.py's 1080p workload.

1. End to end: the same streams decoded with EDGE264_SKIP_NONE, _NONREF and _NONKEY, alternating, `--runs` times each.
   Every stream is decoded by its own decoder (n_threads 0) with the README loop; one Python thread per CPU takes streams
   from a queue (ctypes releases the GIL during the calls).  Decoded frames per second = frames output / wall time; input
   pictures per second = pictures in the streams / wall time (the rate at which the stream is consumed).
2. Host time per mode, in a process of its own per mode with E264_HOST_PROFILE=1 (the decoder's own accounting, printed
   when a decoder is freed): the streams decoded one after another, and the time spent parsing slice data and in the
   other host stages it reports.

It needs a CUDA device and fails without one.  It reads `nvidia-smi --query-gpu` and changes no device setting.

  python tools/skip_cost.py --out results/h100_skip_cost_1080p.txt
"""
import argparse, ctypes, errno, os, queue, re, subprocess, sys, tempfile, threading, time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import edge264_b200 as pkg  # noqa: E402

GEN = "--gop IPB --idr 30 --refs 2 --t8x8 50 --deblock 0 --density 52 --qp 28 --wp 0"   # bench.py CONFIGS["1080p"]
MODES = [("none", pkg.SKIP_NONE), ("nonref", pkg.SKIP_NONREF), ("nonkey", pkg.SKIP_NONKEY)]


def streams(n, frames, workdir):
    """bench.py's streams (same seeds), written in parallel"""
    paths = [os.path.join(workdir, "120x68_%d_%d.264" % (s, frames)) for s in range(2000, 2000 + n)]
    procs = [subprocess.Popen([os.path.join(ROOT, "tools", "gen264"), "-o", p, "-W", "120", "-H", "68", "-n", str(frames), "-s", str(2000 + k)] + GEN.split(),
                              stderr=subprocess.DEVNULL) for k, p in enumerate(paths)]
    if any(q.wait() for q in procs):
        raise RuntimeError("gen264 failed")
    return paths


def decode_one(lib, data, skip):
    buf = ctypes.create_string_buffer(data, len(data) + 64)
    base = ctypes.addressof(buf); end = base + len(data)
    dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
    if not dec:
        raise RuntimeError("edge264_alloc failed (no CUDA device: the GPU backend has no CPU fallback)")
    if lib.edge264_set_skip(dec, skip):
        raise RuntimeError("edge264_set_skip failed")
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


def e2e(lib, bufs, skip, threads):
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
            counts.append(decode_one(lib, b, skip))
    t0 = time.perf_counter()
    th = [threading.Thread(target=work) for _ in range(threads)]
    for t in th: t.start()
    for t in th: t.join()
    return sum(counts), time.perf_counter() - t0


def host_profile(paths, skip):
    """E264_HOST_PROFILE=1 in a child process (the decoder reads it once per process): {stage: (ms total, calls)}"""
    code = ("import sys; sys.path[:0] = [%r, %r]; import skip_cost as s, edge264_b200 as pkg; lib = pkg.load(); "
            "[s.decode_one(lib, open(p, 'rb').read(), %d) for p in sys.argv[1:]]" % (ROOT, os.path.join(ROOT, "tools"), skip))
    r = subprocess.run([sys.executable, "-c", code] + paths, capture_output=True, text=True, timeout=1800,
                       env=dict(os.environ, E264_HOST_PROFILE="1"))
    if r.returncode:
        raise RuntimeError(r.stderr[-2000:])
    out = {}
    for m in re.finditer(r"host profile: (\S+)\s+([\d.]+) ms total\s+(\d+) calls", r.stderr):
        t, n = out.get(m.group(1), (0.0, 0))
        out[m.group(1)] = (t + float(m.group(2)), n + int(m.group(3)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=32); ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--runs", type=int, default=3); ap.add_argument("--threads", type=int, default=len(os.sched_getaffinity(0)))
    ap.add_argument("--profile-streams", type=int, default=4); ap.add_argument("--out", required=True)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("skip_cost.py measures on a CUDA device; none is available")
    lines = []
    def say(s):
        print(s, flush=True); lines.append(s)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    say("card: %s (name, power limit; read in this run)" % card.splitlines()[0] if card else "card: nvidia-smi gave nothing")
    lib = pkg.load()
    paths = streams(a.streams, a.frames, tempfile.mkdtemp(prefix="e264_skip_cost"))
    bufs = [open(p, "rb").read() for p in paths]
    pictures = a.streams * a.frames
    say("workload: %d streams x %d frames, 1920x1088 (%s), %d host threads, one decoder per stream (n_threads 0)" % (len(bufs), a.frames, GEN, a.threads))
    for _, skip in MODES:        # warm-up: device contexts, pinned buffers, code pages
        e2e(lib, bufs[:a.threads], skip, a.threads)
    res = {m: [] for m, _ in MODES}
    for r in range(a.runs):
        for m, skip in MODES:
            n, dt = e2e(lib, bufs, skip, a.threads)
            res[m].append((n / dt, pictures / dt))
            say("run %d skip %-6s  %5d frames out of %d pictures in %.3f s  %.1f decoded frames/s  %.1f input pictures/s" % (r + 1, m, n, pictures, dt, n / dt, pictures / dt))
    for m, _ in MODES:
        fr = sorted(v[0] for v in res[m]); pi = sorted(v[1] for v in res[m])
        say("skip %-6s  decoded frames/s median %.1f (min %.1f, max %.1f)  input pictures/s median %.1f (min %.1f, max %.1f)"
            % (m, fr[len(fr) // 2], fr[0], fr[-1], pi[len(pi) // 2], pi[0], pi[-1]))
    for m, skip in MODES:
        prof = host_profile(paths[:a.profile_streams], skip)
        n_pics = a.profile_streams * a.frames
        say("host profile, skip %s, %d streams one after another (%d input pictures):" % (m, a.profile_streams, n_pics))
        for k in sorted(prof):
            t, n = prof[k]
            say("  %-18s %9.1f ms total  %6d calls  %7.1f us per input picture" % (k, t, n, 1e3 * t / n_pics))
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fo:
        fo.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
