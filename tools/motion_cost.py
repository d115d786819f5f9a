"""What the motion export (include/edge264_motion.h) costs on the GPU, on bench.py's 1080p workload.

1. End to end: the same streams decoded with the export off and on, alternating, `--runs` times each.  Every stream is
   decoded by its own decoder (n_threads 0) with the README loop; one Python thread per CPU takes streams from a queue
   (ctypes releases the GIL during the calls).  Frames per second = frames decoded / wall time.
2. In a separate run, torch.profiler with CUDA activities over a few streams decoded with the export on: the device time
   per picture of e264_motion_kernel next to the reconstruction kernels.

  python tools/motion_cost.py --out results/h100_motion_cost_1080p.txt
"""
import argparse, ctypes, errno, os, queue, subprocess, sys, tempfile, threading, time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import edge264_b200 as pkg  # noqa: E402

GEN = "--gop IPB --idr 30 --refs 2 --t8x8 50 --deblock 0 --density 52 --qp 28 --wp 0"   # bench.py CONFIGS["1080p"]


def streams(n, frames, workdir):
    """bench.py's streams (same seeds), written in parallel"""
    paths = [os.path.join(workdir, "120x68_%d_%d.264" % (s, frames)) for s in range(2000, 2000 + n)]
    procs = [subprocess.Popen([os.path.join(ROOT, "tools", "gen264"), "-o", p, "-W", "120", "-H", "68", "-n", str(frames), "-s", str(2000 + k)] + GEN.split(),
                              stderr=subprocess.DEVNULL) for k, p in enumerate(paths)]
    if any(q.wait() for q in procs):
        raise RuntimeError("gen264 failed")
    return [open(p, "rb").read() for p in paths]


def decode_one(lib, data, motion):
    buf = ctypes.create_string_buffer(data, len(data) + 64)
    base = ctypes.addressof(buf); end = base + len(data)
    dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
    if motion and lib.edge264_enable_motion(dec):
        raise RuntimeError("edge264_enable_motion failed")
    nal, n, f, m = base + 3 + (1 if data[2] == 0 else 0), 0, pkg.Edge264Frame(), pkg.Edge264Motion()
    while True:
        sc = lib.edge264_find_start_code(nal, end, 0) if nal < end else end
        res = lib.edge264_decode_NAL(dec, nal, sc, None, None)
        while lib.edge264_get_frame(dec, ctypes.byref(f), 0) == 0:
            n += 1
            if motion and lib.edge264_get_motion(dec, ctypes.byref(f), ctypes.byref(m)):
                raise RuntimeError("edge264_get_motion failed")
        if res == errno.ENOBUFS:
            continue
        if nal >= end:
            break
        nal = sc + 3 if sc + 3 < end else end
    d = ctypes.c_void_p(dec)
    lib.edge264_free(ctypes.byref(d))
    return n


def e2e(lib, bufs, motion, threads):
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
            counts.append(decode_one(lib, b, motion))
    t0 = time.perf_counter()
    th = [threading.Thread(target=work) for _ in range(threads)]
    for t in th: t.start()
    for t in th: t.join()
    return sum(counts), time.perf_counter() - t0


def profile(lib, bufs):
    import torch
    from torch.profiler import profile as tprof, ProfilerActivity
    torch.cuda.init()
    with tprof(activities=[ProfilerActivity.CUDA]) as p:
        frames = sum(decode_one(lib, b, True) for b in bufs)
        torch.cuda.synchronize()
    per = {}
    for e in p.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:   # kernels and copies, with their device time
            per.setdefault(e.name.split("(")[0], []).append(e.time_range.elapsed_us())
    return frames, per


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=32); ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--runs", type=int, default=3); ap.add_argument("--threads", type=int, default=len(os.sched_getaffinity(0)))
    ap.add_argument("--profile-streams", type=int, default=2); ap.add_argument("--out", required=True)
    a = ap.parse_args()
    lines = []
    def say(s):
        print(s, flush=True); lines.append(s)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    say("card: %s (name, power limit; read in this run)" % card.splitlines()[0] if card else "card: nvidia-smi gave nothing")
    lib = pkg.load()
    bufs = streams(a.streams, a.frames, tempfile.mkdtemp(prefix="e264_motion_cost"))
    say("workload: %d streams x %d frames, 1920x1088 (%s), %d host threads, one decoder per stream (n_threads 0)" % (len(bufs), a.frames, GEN, a.threads))
    e2e(lib, bufs[:a.threads], False, a.threads)       # warm-up: device contexts, pinned buffers, code pages
    e2e(lib, bufs[:a.threads], True, a.threads)
    res = {False: [], True: []}
    for r in range(a.runs):
        for motion in (False, True):
            n, dt = e2e(lib, bufs, motion, a.threads)
            res[motion].append(n / dt)
            say("run %d export %-3s  %d frames in %.3f s  %.1f frames/s" % (r + 1, "on" if motion else "off", n, dt, n / dt))
    for motion in (False, True):
        v = sorted(res[motion])
        say("export %-3s  median %.1f frames/s (min %.1f, max %.1f)" % ("on" if motion else "off", v[len(v) // 2], v[0], v[-1]))
    frames, per = profile(lib, bufs[:a.profile_streams])
    say("torch.profiler, %d streams with the export on (%d pictures): device time per launch, us" % (a.profile_streams, frames))
    for k in sorted(per):
        v = per[k]
        say("  %-60s launches %5d  mean %8.2f  total per picture %8.2f" % (k, len(v), sum(v) / len(v), sum(v) / frames))
    with open(a.out, "w") as fo:
        fo.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
