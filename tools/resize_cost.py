"""What the resized output (include/edge264_packed.h, edge264_enable_resized) costs on the GPU, on bench.py's 1080p workload.

1. End to end: the same streams decoded with the resized output off, as NV12 at 1280x720 and as NV12 at 224x224,
   alternating, `--runs` times each.  Every stream is decoded by its own decoder (n_threads 0)
   with the README loop; one Python thread per CPU takes streams from a queue (ctypes releases the GIL during the calls).
   Frames per second = frames decoded / wall time.
2. In a separate pass per mode, torch.profiler with CUDA activities over a few streams: the device time per picture of
   e264_resize_kernel and of the copies next to the reconstruction kernels, and the kernel's achieved bytes per second
   from the bytes the definition needs (the cropped picture read once, the resized planes written once).

It needs a CUDA device and fails without one.  It reads `nvidia-smi --query-gpu` and changes no device setting.

  python tools/resize_cost.py --out results/h100_resize_cost_1080p.txt
"""
import argparse, ctypes, errno, os, queue, subprocess, sys, tempfile, threading, time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import edge264_b200 as pkg  # noqa: E402

GEN = "--gop IPB --idr 30 --refs 2 --t8x8 50 --deblock 0 --density 52 --qp 28 --wp 0"   # bench.py CONFIGS["1080p"]
W, H = 1920, 1088
MODES = [("off", None), ("nv12 1280x720", (pkg.PACKED_NV12, 1280, 720)), ("nv12 224x224", (pkg.PACKED_NV12, 224, 224))]
HBM_PEAK = 3.35e12   # bytes/s, H100 SXM data sheet


def streams(n, frames, workdir):
    """bench.py's streams (same seeds), written in parallel"""
    paths = [os.path.join(workdir, "120x68_%d_%d.264" % (s, frames)) for s in range(2000, 2000 + n)]
    procs = [subprocess.Popen([os.path.join(ROOT, "tools", "gen264"), "-o", p, "-W", "120", "-H", "68", "-n", str(frames), "-s", str(2000 + k)] + GEN.split(),
                              stderr=subprocess.DEVNULL) for k, p in enumerate(paths)]
    if any(q.wait() for q in procs):
        raise RuntimeError("gen264 failed")
    return [open(p, "rb").read() for p in paths]


def decode_one(lib, data, resized):
    buf = ctypes.create_string_buffer(data, len(data) + 64)
    base = ctypes.addressof(buf); end = base + len(data)
    dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
    if not dec:
        raise RuntimeError("edge264_alloc failed (no CUDA device: the GPU backend has no CPU fallback)")
    if resized is not None and lib.edge264_enable_resized(dec, *resized):
        raise RuntimeError("edge264_enable_resized failed")
    nal, n, f, p = base + 3 + (1 if data[2] == 0 else 0), 0, pkg.Edge264Frame(), pkg.Edge264Packed()
    while True:
        sc = lib.edge264_find_start_code(nal, end, 0) if nal < end else end
        res = lib.edge264_decode_NAL(dec, nal, sc, None, None)
        while lib.edge264_get_frame(dec, ctypes.byref(f), 0) == 0:
            n += 1
            if resized is not None and lib.edge264_get_packed(dec, ctypes.byref(f), ctypes.byref(p)):
                raise RuntimeError("edge264_get_packed failed")
        if res == errno.ENOBUFS:
            continue
        if nal >= end:
            break
        nal = sc + 3 if sc + 3 < end else end
    d = ctypes.c_void_p(dec)
    lib.edge264_free(ctypes.byref(d))
    return n


def e2e(lib, bufs, resized, threads):
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
            counts.append(decode_one(lib, b, resized))
    t0 = time.perf_counter()
    th = [threading.Thread(target=work) for _ in range(threads)]
    for t in th: t.start()
    for t in th: t.join()
    return sum(counts), time.perf_counter() - t0


def profile(lib, bufs, resized):
    import torch
    from torch.profiler import profile as tprof, ProfilerActivity
    with tprof(activities=[ProfilerActivity.CUDA]) as p:
        frames = sum(decode_one(lib, b, resized) for b in bufs)
        torch.cuda.synchronize()
    per = {}
    for e in p.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:   # kernels and copies, with their device time
            name = e.name.split("(")[0]
            per.setdefault(name[5:] if name.startswith("void ") else name, []).append(e.time_range.elapsed_us())
    return frames, per


def definition_bytes(resized):
    """bytes the definition needs per picture: the cropped planes read once, the resized samples written once (no padding)"""
    return W * H * 3 // 2, resized[1] * resized[2] * 3 // 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=32); ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--runs", type=int, default=3); ap.add_argument("--threads", type=int, default=len(os.sched_getaffinity(0)))
    ap.add_argument("--profile-streams", type=int, default=2); ap.add_argument("--out", required=True)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("resize_cost.py measures on a CUDA device; none is available")
    torch.cuda.init()
    lines = []
    def say(s):
        print(s, flush=True); lines.append(s)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    say("card: %s (name, power limit; read in this run)" % card.splitlines()[0] if card else "card: nvidia-smi gave nothing")
    lib = pkg.load()
    bufs = streams(a.streams, a.frames, tempfile.mkdtemp(prefix="e264_resize_cost"))
    say("workload: %d streams x %d frames, %dx%d (%s), %d host threads, one decoder per stream (n_threads 0)" % (len(bufs), a.frames, W, H, GEN, a.threads))
    for _, resized in MODES:       # warm-up: device contexts, pinned buffers, code pages
        e2e(lib, bufs[:a.threads], resized, a.threads)
    res = {m: [] for m, _ in MODES}
    for r in range(a.runs):
        for m, resized in MODES:
            n, dt = e2e(lib, bufs, resized, a.threads)
            res[m].append(n / dt)
            say("run %d resized %-14s  %d frames in %.3f s  %.1f frames/s" % (r + 1, m, n, dt, n / dt))
    for m, _ in MODES:
        v = sorted(res[m])
        say("resized %-14s  median %.1f frames/s (min %.1f, max %.1f)" % (m, v[len(v) // 2], v[0], v[-1]))
    for m, resized in MODES:
        frames, per = profile(lib, bufs[:a.profile_streams], resized)
        say("torch.profiler, %d streams, resized %s (%d pictures): device time per launch, us" % (a.profile_streams, m, frames))
        for k in sorted(per):
            v = per[k]
            say("  %-60s launches %5d  mean %8.2f  total per picture %8.2f" % (k, len(v), sum(v) / len(v), sum(v) / frames))
        pk = [v for k, v in per.items() if k.startswith("e264_resize_kernel")]
        if resized is not None:
            if len(pk) != 1 or len(pk[0]) != frames:
                raise SystemExit("expected one e264_resize_kernel launch per picture")
            rd, wr = definition_bytes(resized)
            us = sum(pk[0]) / frames
            rate = (rd + wr) / (us * 1e-6)
            say("  e264_resize_kernel (kernel figure): %d bytes read + %d written per picture in %.2f us = %.0f GB/s, %.1f %% of the data sheet's 3.35 TB/s; "
                "floor at that bandwidth %.2f us" % (rd, wr, us, rate / 1e9, 100 * rate / HBM_PEAK, (rd + wr) / HBM_PEAK * 1e6))
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fo:
        fo.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
