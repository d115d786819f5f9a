"""How long low-latency output (include/edge264_latency.h, edge264_set_output_latency) holds frames, against the default
decoder, on 1080p streams.

For every frame: the host-clock time from the edge264_decode_NAL call that completed its picture (the call passing the
picture's last NAL unit) to the edge264_get_frame call that returned it, and the number of pictures whose first NAL unit
was passed in between (the frames it was held for).  Cases:
  - streams: 1080p IPPP at level 5.1 without VUI (tools/gen264 --no-vui: the level gives a reorder depth of 16, the case of
    many cameras), decoded with depth 0; bench.py's 1080p IPB streams (VUI reorder depth 1), decoded with depth 1;
  - the default decoder against the mode; 0 and 3 parse-ahead threads; colour and luma-only;
  - one stream at a time with its pictures passed in at 30 fps (a live source), and 16 streams at once, unpaced, one
    host thread each, for throughput.
The card's name and power limit are read in the same run.  It needs a CUDA device and fails without one; it reads
`nvidia-smi --query-gpu` and changes no device setting.

  python tools/latency_cost.py --out results/h100_latency_1080p.txt
"""
import argparse, ctypes, errno, os, subprocess, sys, tempfile, threading, time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import edge264_b200 as pkg  # noqa: E402

IPPP = dict(bench.CONFIGS["1080p"], gen="--gop IP --idr 30 --refs 2 --t8x8 50 --deblock 0 --density 52 --qp 28 --wp 0 --level 51 --no-vui")
STREAMS = [("1080p IPPP, no VUI, level 5.1", IPPP, 0), ("bench.py 1080p IPB", bench.CONFIGS["1080p"], 1)]


def nal_units(data):
    """(start, end) of every NAL unit and, per NAL unit, the index of the picture it belongs to (a picture starts with a
    parameter set or the slice of first_mb_in_slice 0 that follows the previous picture's slices)"""
    starts, i = [], 0
    while (j := data.find(b"\x00\x00\x01", i)) >= 0:
        starts.append(j + 3); i = j + 3
    nals = [(s, (starts[k + 1] - 3 if k + 1 < len(starts) else len(data))) for k, s in enumerate(starts)]
    pic, seen_slice, owner = 0, False, []
    for s, _ in nals:
        t = data[s] & 31
        first = t in (1, 5) and data[s + 1] & 0x80
        if seen_slice and (first or t in (7, 8)):
            pic += 1; seen_slice = False
        seen_slice |= t in (1, 5)
        owner.append(pic)
    return nals, owner


def decode(lib, data, latency, threads, luma, fps):
    """One decode with the README loop; fps > 0 passes picture k's NAL units in at k / fps seconds.  Per frame (latency in
    seconds, pictures started in between); and the wall time."""
    nals, owner = nal_units(data)
    last = {p: k for k, p in enumerate(owner)}
    buf = ctypes.create_string_buffer(data, len(data) + 64)
    base = ctypes.addressof(buf)
    dec = lib.edge264_alloc(threads, None, None, 0, None, None, None)
    if not dec:
        raise RuntimeError("edge264_alloc failed (no CUDA device: the GPU backend has no CPU fallback)")
    if luma and lib.edge264_enable_luma_only(dec):
        raise RuntimeError("edge264_enable_luma_only failed")
    if lib.edge264_set_output_latency(dec, latency):
        raise RuntimeError("edge264_set_output_latency failed")
    done, out, f = {}, [], pkg.Edge264Frame()
    t0 = time.perf_counter()
    k = 0
    while k <= len(nals):
        if k < len(nals):
            if fps and (wait := t0 + owner[k] / fps - time.perf_counter()) > 0:
                time.sleep(wait)
            a, b = nals[k]
            t_call = time.perf_counter()
            res = lib.edge264_decode_NAL(dec, base + a, base + b, None, None)
        else:
            t_call = time.perf_counter()
            res = lib.edge264_decode_NAL(dec, base + len(data), base + len(data), None, None)
        if k < len(nals) and last[owner[k]] == k and res != errno.ENOBUFS:
            done[owner[k]] = t_call
        started = owner[k] + 1 if k < len(nals) else owner[-1] + 1
        while lib.edge264_get_frame(dec, ctypes.byref(f), 0) == 0:
            out.append((f.FrameId, time.perf_counter(), started))
        if res == errno.ENOBUFS:
            continue
        k += 1
    wall = time.perf_counter() - t0
    d = ctypes.c_void_p(dec)
    lib.edge264_free(ctypes.byref(d))
    # FrameIds grow in decoding order (an IDR after other pictures skips some), and every picture is output
    pic = {i: p for p, i in enumerate(sorted(i for i, _, _ in out))}
    return [(t - done[pic[i]], started - pic[i] - 1) for i, t, started in out], wall


def stats(per):
    lat = sorted(x[0] * 1e3 for x in per)
    held = [x[1] for x in per]
    q = lambda v, p: v[min(len(v) - 1, int(p * len(v)))]
    return "held mean %5.2f max %2d | latency ms mean %7.2f p50 %7.2f p95 %7.2f max %7.2f" % (
        sum(held) / len(held), max(held), sum(lat) / len(lat), q(lat, 0.5), q(lat, 0.95), lat[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60); ap.add_argument("--streams", type=int, default=16)
    ap.add_argument("--out", required=True)
    a = ap.parse_args()
    lines = []
    def say(s):
        print(s, flush=True); lines.append(s)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    say("card: %s (name, power limit; read in this run)" % card.splitlines()[0] if card else "card: nvidia-smi gave nothing")
    lib = pkg.load()
    tmp = tempfile.mkdtemp(prefix="e264_latency_cost")
    for title, cfg, depth in STREAMS:
        bufs = bench.generate_streams(cfg, [cfg["seed0"] + i for i in range(a.streams)], a.frames, os.path.join(tmp, str(depth)))
        say("")
        say("%s: %dx%d, %d frames per stream (%s); mode depth %d" % (title, cfg["w"] * 16, cfg["h"] * 16, a.frames, cfg["gen"], depth))
        decode(lib, bufs[0], -1, 0, False, 0)   # warm-up: module load, first allocations
        for luma in (False, True):
            for threads in (0, 3):
                for lat in (-1, depth):
                    label = "%-7s %-10s threads %d" % ("default" if lat < 0 else "depth %d" % lat, "luma-only" if luma else "colour", threads)
                    per, _ = decode(lib, bufs[0], lat, threads, luma, 30.0)
                    say("  one stream at 30 fps   %s: %s" % (label, stats(per)))
                    res = [None] * len(bufs)
                    def work(i):
                        res[i] = decode(lib, bufs[i], lat, threads, luma, 0)
                    t0 = time.perf_counter()
                    th = [threading.Thread(target=work, args=(i,)) for i in range(len(bufs))]
                    for t in th: t.start()
                    for t in th: t.join()
                    wall = time.perf_counter() - t0
                    per = [x for r in res for x in r[0]]
                    say("  %2d streams unpaced    %s: %s | %7.1f frames/s" % (len(bufs), label, stats(per), len(per) / wall))
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fo:
        fo.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
