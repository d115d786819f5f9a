"""What the picture statistics (include/edge264_picstats.h, edge264_enable_picstats) cost on the GPU, on bench.py's 1080p
workload.

1. End to end: the same streams decoded with the statistics off, with them on, and with the same statistics computed by
   numpy from the host frames inside the decode loop (the work the feature replaces), alternating, `--runs` times each.
   Every stream is decoded by its own decoder (n_threads 0) with the README loop; one Python thread per CPU takes streams
   from a queue (ctypes releases the GIL during the calls, numpy during most of its work).  Frames per second = frames
   decoded / wall time.
2. A separate torch.profiler pass with CUDA activities over a few streams: the device time per picture of
   e264_picstats_kernel, its memset and its copy next to the reconstruction kernels, and the kernel's achieved bytes per
   second from the bytes the definition needs (the coded picture read once, the statistics written once).
3. The same profile on constant pictures (constant_stream: I_PCM macroblocks of one value, decoded luma-only, so every
   plane is constant), the histogram's worst case: every sample falls into one bin.

It needs a CUDA device and fails without one.  It reads `nvidia-smi --query-gpu` and changes no device setting.

  python tools/picstats_cost.py --out results/h100_picstats_cost_1080p.txt
"""
import argparse, ctypes, errno, os, queue, subprocess, sys, tempfile, threading, time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import edge264_b200 as pkg  # noqa: E402

GEN = "--gop IPB --idr 30 --refs 2 --t8x8 50 --deblock 0 --density 52 --qp 28 --wp 0"   # bench.py CONFIGS["1080p"]
W, H = 1920, 1088
MODES = ["off", "on", "numpy"]
HBM_PEAK = 3.35e12   # bytes/s, H100 SXM data sheet


def constant_stream(w_mbs, h_mbs, frames, value, crop_bottom=0):
    """An Annex-B stream of `frames` IDR pictures whose macroblocks are all I_PCM with every sample equal to `value`
    (4..255): Main profile, CAVLC, deblocking off, POC type 2.  It decodes to constant planes."""
    assert 4 <= value <= 255 and not crop_bottom & 1
    def rbsp(fields):
        bits = []
        for kind, v in fields:
            if kind == "ue" or kind == "se":
                v = (2 * v - 1 if v > 0 else -2 * v) if kind == "se" else v
                n = (v + 1).bit_length()
                bits += [0] * (n - 1) + [(v + 1) >> (n - 1 - i) & 1 for i in range(n)]
            else:
                bits += [v >> (kind - 1 - i) & 1 for i in range(kind)]
        bits += [0] * (-len(bits) % 8)
        return bytes(int("".join(map(str, bits[i:i + 8])), 2) for i in range(0, len(bits), 8))
    def nal(header, payload, samples=b""):
        out, zeros = bytearray(), 0
        for b in payload:                       # emulation prevention; the samples and their mb_type words never need it
            if zeros >= 2 and b <= 3:
                out.append(3); zeros = 0
            out.append(b); zeros = zeros + 1 if b == 0 else 0
        return b"\x00\x00\x00\x01" + bytes([header]) + bytes(out) + samples
    level = 40 if w_mbs * h_mbs <= 8192 else 62
    crop = [(1, 1), ("ue", 0), ("ue", 0), ("ue", 0), ("ue", crop_bottom // 2)] if crop_bottom else [(1, 0)]
    sps = [(8, 77), (8, 0), (8, level), ("ue", 0), ("ue", 0), ("ue", 2), ("ue", 1), (1, 0), ("ue", w_mbs - 1), ("ue", h_mbs - 1), (1, 1), (1, 1)] + crop + [(1, 0), (1, 1)]
    pps = [("ue", 0), ("ue", 0), (1, 0), (1, 0), ("ue", 0), ("ue", 0), ("ue", 0), (1, 0), (2, 0), ("se", 0), ("se", 0), ("se", 0), (1, 1), (1, 0), (1, 0), (1, 1)]
    pcm = b"\x0d\x00" + bytes([value]) * 384    # mb_type ue(25) = I_PCM, pcm_alignment_zero_bits, 256 + 2 x 64 samples
    out = nal(0x67, rbsp(sps)) + nal(0x68, rbsp(pps))
    for k in range(frames):
        head = rbsp([("ue", 0), ("ue", 7), ("ue", 0), (4, 0), ("ue", k & 1), (1, 0), (1, 0), ("se", 0), ("ue", 1), ("ue", 25)])
        out += nal(0x65, head, pcm[2:] + pcm * (w_mbs * h_mbs - 1) + b"\x80")
    return out


def streams(n, frames, workdir):
    """bench.py's streams (same seeds), written in parallel"""
    paths = [os.path.join(workdir, "120x68_%d_%d.264" % (s, frames)) for s in range(2000, 2000 + n)]
    procs = [subprocess.Popen([os.path.join(ROOT, "tools", "gen264"), "-o", p, "-W", "120", "-H", "68", "-n", str(frames), "-s", str(2000 + k)] + GEN.split(),
                              stderr=subprocess.DEVNULL) for k, p in enumerate(paths)]
    if any(q.wait() for q in procs):
        raise RuntimeError("gen264 failed")
    return [open(p, "rb").read() for p in paths]


def numpy_stats(f):
    """the definition over a host frame: histograms of the cropped planes, sums and sums of squares per coded macroblock"""
    import numpy as np
    top, right, bottom, left = f.frame_crop_offsets
    out = []
    for p in range(3):
        n, s = (8, 1) if p else (16, 0)
        w, h, st = (f.width_C, f.height_C, f.stride_C) if p else (f.width_Y, f.height_Y, f.stride_Y)
        cw, ch = w + ((left + right) >> s), h + ((top + bottom) >> s)
        base = ctypes.cast(f.samples[p], ctypes.c_void_p).value - (top >> s) * st - (left >> s)
        plane = np.lib.stride_tricks.as_strided(np.frombuffer(ctypes.string_at(base, (ch - 1) * st + cw), np.uint8), (ch, cw), (st, 1))
        v = plane.astype(np.uint32).reshape(ch // n, n, cw // n, n)
        out.append((np.bincount(plane[top >> s:(top >> s) + h, left >> s:(left >> s) + w].ravel(), minlength=256), v.sum(axis=(1, 3)), (v * v).sum(axis=(1, 3))))
    return out


def decode_one(lib, data, mode, luma_only=False):
    buf = ctypes.create_string_buffer(data, len(data) + 64)
    base = ctypes.addressof(buf); end = base + len(data)
    dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
    if not dec:
        raise RuntimeError("edge264_alloc failed (no CUDA device: the GPU backend has no CPU fallback)")
    if mode == "on" and lib.edge264_enable_picstats(dec):
        raise RuntimeError("edge264_enable_picstats failed")
    if luma_only and lib.edge264_enable_luma_only(dec):
        raise RuntimeError("edge264_enable_luma_only failed")
    nal, n, f, s = base + 3 + (1 if data[2] == 0 else 0), 0, pkg.Edge264Frame(), pkg.Edge264PicStats()
    while True:
        sc = lib.edge264_find_start_code(nal, end, 0) if nal < end else end
        res = lib.edge264_decode_NAL(dec, nal, sc, None, None)
        while lib.edge264_get_frame(dec, ctypes.byref(f), 0) == 0:
            n += 1
            if mode == "on" and lib.edge264_get_picstats(dec, ctypes.byref(f), ctypes.byref(s)):
                raise RuntimeError("edge264_get_picstats failed")
            if mode == "numpy":
                numpy_stats(f)
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


def profile(lib, bufs, mode, luma_only=False):
    import torch
    from torch.profiler import profile as tprof, ProfilerActivity
    with tprof(activities=[ProfilerActivity.CUDA]) as p:
        frames = sum(decode_one(lib, b, mode, luma_only) for b in bufs)
        torch.cuda.synchronize()
    per = {}
    for e in p.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:   # kernels and copies, with their device time
            name = e.name.split("(")[0]
            per.setdefault(name[5:] if name.startswith("void ") else name, []).append(e.time_range.elapsed_us())
    return frames, per


def report(say, label, frames, per, nmb):
    say("torch.profiler, %s (%d pictures): device time per launch, us" % (label, frames))
    for k in sorted(per):
        v = per[k]
        say("  %-60s launches %5d  mean %8.2f  total per picture %8.2f" % (k, len(v), sum(v) / len(v), sum(v) / frames))
    ps = [v for k, v in per.items() if k.startswith("e264_picstats_kernel")]
    if len(ps) != 1 or len(ps[0]) != frames:
        raise SystemExit("expected one e264_picstats_kernel launch per picture")
    rd, wr = nmb * 384, 3072 + 24 * nmb
    us = sum(ps[0]) / frames
    rate = (rd + wr) / (us * 1e-6)
    say("  e264_picstats_kernel (kernel figure): %d bytes read + %d written per picture in %.2f us = %.0f GB/s, %.1f %% of the data sheet's 3.35 TB/s; "
        "floor at that bandwidth %.2f us" % (rd, wr, us, rate / 1e9, 100 * rate / HBM_PEAK, (rd + wr) / HBM_PEAK * 1e6))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=32); ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--runs", type=int, default=3); ap.add_argument("--threads", type=int, default=len(os.sched_getaffinity(0)))
    ap.add_argument("--profile-streams", type=int, default=2); ap.add_argument("--out", required=True)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("picstats_cost.py measures on a CUDA device; none is available")
    torch.cuda.init()
    lines = []
    def say(s):
        print(s, flush=True); lines.append(s)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    say("card: %s (name, power limit; read in this run)" % card.splitlines()[0] if card else "card: nvidia-smi gave nothing")
    lib = pkg.load()
    bufs = streams(a.streams, a.frames, tempfile.mkdtemp(prefix="e264_picstats_cost"))
    say("workload: %d streams x %d frames, %dx%d (%s), %d host threads, one decoder per stream (n_threads 0)" % (len(bufs), a.frames, W, H, GEN, a.threads))
    for m in MODES:       # warm-up: device contexts, pinned buffers, code pages
        e2e(lib, bufs[:a.threads], m, a.threads)
    res = {m: [] for m in MODES}
    for r in range(a.runs):
        for m in MODES:
            n, dt = e2e(lib, bufs, m, a.threads)
            res[m].append(n / dt)
            say("run %d picstats %-6s  %d frames in %.3f s  %.1f frames/s" % (r + 1, m, n, dt, n / dt))
    for m in MODES:
        v = sorted(res[m])
        say("picstats %-6s  median %.1f frames/s (min %.1f, max %.1f)" % (m, v[len(v) // 2], v[0], v[-1]))
    nmb = (W // 16) * (H // 16)
    frames, per = profile(lib, bufs[:a.profile_streams], "on")
    report(say, "%d streams, picstats on" % a.profile_streams, frames, per, nmb)
    # the worst case of the histogram: constant planes (checked here before they are profiled)
    const = constant_stream(W // 16, H // 16, 30, 77, crop_bottom=8)
    frames_c = pkg.decode_bytes(const, lib, luma_only=True, picstats=True)[0]
    for f in frames_c:
        h = f[-1]["hist"]
        if not (h[0][77] == 1920 * 1080 and h[1][128] == h[2][128] == 960 * 540 and f[3] == bytes([77]) * 1920 * 1080 + bytes([128]) * 960 * 1080):
            raise SystemExit("the constant stream did not decode to constant planes")
    say("constant pictures: %d frames, Y all 77, Cb and Cr all 128 (luma-only), checked on the decoded samples and the histograms" % len(frames_c))
    frames, per = profile(lib, [const] * a.profile_streams, "on", luma_only=True)
    report(say, "%d constant streams, luma-only, picstats on" % a.profile_streams, frames, per, nmb)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fo:
        fo.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
