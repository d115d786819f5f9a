"""What decoding the second view of a stereo stream (include/edge264_mvc.h) costs on the GPU: 1080p stereo IPB streams
(bench.py's 1080p generator arguments with tools/gen264 --mvc) against the same streams with their prefix NAL units,
subset SPSs and second-view slices (NAL unit types 14, 15, 20) removed, which decode to the same base views.

1. Kernel-only replay: every stream decoded once with the README loop (one decoder per stream, n_threads 0, records kept
   with E264B_KEEP=1); then e264b_replay of the stereo and the single-view decoders, alternating, `--runs` times each.
   Device time per access unit (one picture single-view, two stereo) and the ratio of the two.
2. Host-to-device and device-to-host bytes and kernel launches per access unit (e264b_stats) of the decodes of step 1.
3. The card's name and power limit, read in the same run.

It needs a CUDA device and fails without one.  It reads `nvidia-smi --query-gpu` and changes no device setting.

  python tools/mvc_cost.py --out results/h100_mvc_cost_1080p.txt
"""
import argparse, ctypes, errno, os, subprocess, sys, tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import edge264_b200 as pkg  # noqa: E402


def strip_mvc(data):
    """The stream without its NAL units of types 14, 15 and 20."""
    out, starts, i = [], [], 0
    while (j := data.find(b"\x00\x00\x01", i)) >= 0:
        starts.append(j + 3); i = j + 3
    for k, s in enumerate(starts):
        e = starts[k + 1] - 3 if k + 1 < len(starts) else len(data)
        if data[s] & 31 not in (14, 15, 20):
            out.append(b"\x00\x00\x00\x01" + data[s:e].rstrip(b"\x00") if k + 1 < len(starts) else b"\x00\x00\x00\x01" + data[s:e])
    return b"".join(out)


def decode_keep(lib, data):
    """The README loop; returns (decoder, access units output).  The decoder is left allocated: its device context keeps
    the records for the replay."""
    buf = ctypes.create_string_buffer(data, len(data) + 64)
    base = ctypes.addressof(buf); end = base + len(data)
    dec = lib.edge264_alloc(0, None, None, 0, None, None, None)
    if not dec:
        raise RuntimeError("edge264_alloc failed (no CUDA device: the GPU backend has no CPU fallback)")
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
    return dec, n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=16); ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--replay-steps", type=int, default=3); ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", required=True)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("mvc_cost.py measures on a CUDA device; none is available")
    lines = []
    def say(s):
        print(s, flush=True); lines.append(s)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    say("card: %s (name, power limit; read in this run)" % card.splitlines()[0] if card else "card: nvidia-smi gave nothing")
    cfg = bench.CONFIGS["1080p"]
    tmp = tempfile.mkdtemp(prefix="e264_mvc_cost")
    stereo = []
    for i in range(a.streams):
        path = os.path.join(tmp, "s%d.264" % i)
        seed = cfg["seed0"] + i
        subprocess.run([os.path.join(ROOT, "tools", "gen264"), "-o", path, "-W", str(cfg["w"]), "-H", str(cfg["h"]), "-n", str(a.frames), "-s", str(seed)]
                       + cfg["gen"].split() + ["--mvc", str(seed)], check=True, stderr=subprocess.DEVNULL)
        stereo.append(open(path, "rb").read())
    sets = {"stereo": stereo, "single": [strip_mvc(d) for d in stereo]}
    say("workload: %d streams x %d access units, %dx%d (%s --mvc), and the same streams without NAL units 14/15/20" % (a.streams, a.frames, cfg["w"] * 16, cfg["h"] * 16, cfg["gen"]))
    lib = pkg.load()
    core = ctypes.CDLL(pkg.LIB_PATH)
    core.e264b_of_decoder.restype = ctypes.c_void_p; core.e264b_of_decoder.argtypes = [ctypes.c_void_p]
    core.e264b_replay.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.POINTER(bench.ReplayStats)]
    core.e264b_stats.argtypes = [ctypes.c_void_p] + [ctypes.POINTER(ctypes.c_uint64)] * 3
    core.e264b_error_flag.argtypes = [ctypes.c_void_p]
    core.e264b_kept_count.argtypes = [ctypes.c_void_p]

    os.environ["E264B_KEEP"] = "1"
    kept = {}
    for name, bufs in sets.items():
        decoded = [decode_keep(lib, d) for d in bufs]
        devs = (ctypes.c_void_p * len(bufs))(*[core.e264b_of_decoder(d) for d, _ in decoded])
        aus = sum(n for _, n in decoded)
        tot = [0, 0, 0]
        for i in range(len(bufs)):
            v = [ctypes.c_uint64() for _ in range(3)]
            core.e264b_stats(devs[i], *[ctypes.byref(x) for x in v])
            tot = [t + x.value for t, x in zip(tot, v)]
        pics = sum(core.e264b_kept_count(devs[i]) for i in range(len(bufs)))
        say("counts %-7s %d access units, %d pictures: kernel launches %.2f, host-to-device %.0f bytes, device-to-host %.0f bytes per access unit"
            % (name, aus, pics, tot[0] / aus, tot[1] / aus, tot[2] / aus))
        kept[name] = ([d for d, _ in decoded], devs, aus)
    os.environ["E264B_KEEP"] = "0"
    S, T = a.streams, 8
    for name in sets:     # warm-up: module loads
        st = bench.ReplayStats()
        if core.e264b_replay(kept[name][1], S, 1, T, ctypes.byref(st)):
            raise SystemExit("e264b_replay failed")
    per_au = {name: [] for name in sets}
    for r in range(a.runs):
        for name in sets:
            _, devs, aus = kept[name]
            st = bench.ReplayStats()
            if core.e264b_replay(devs, S, a.replay_steps, T, ctypes.byref(st)) or any(core.e264b_error_flag(devs[i]) for i in range(S)):
                raise SystemExit("e264b_replay failed")
            us = 1000 * st.ms_total / (aus * a.replay_steps)
            per_au[name].append(us)
            spans = " ".join("%s %.0f us" % (k, 1000 * st.kernel_ms[i] / max(1, st.kernel_launches[i])) for i, k in ((1, "inter"), (2, "intra"), (3, "deblock")))
            say("replay run %d %-7s %d streams in flight: %.1f ms per step, %.2f us of device time per access unit; mean span per launch: %s"
                % (r + 1, name, S, st.ms_total / a.replay_steps, us, spans))
    med = {name: sorted(v)[len(v) // 2] for name, v in per_au.items()}
    for name, v in per_au.items():
        say("replay %-7s median %.2f us per access unit (min %.2f, max %.2f)" % (name, med[name], min(v), max(v)))
    say("stereo / single-view device time per access unit: %.2f" % (med["stereo"] / med["single"]))
    for name in sets:
        for d in kept[name][0]:
            p = ctypes.c_void_p(d)
            lib.edge264_free(ctypes.byref(p))
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fo:
        fo.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
