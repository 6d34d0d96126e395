"""Where C2's time goes: the fused sweep kernel set against the streaming ceiling of the GPU it runs on.

Reports, at 2^26 fp32 elements, the best kernel time (CUDA events around each launch) of
  (a) ceiling  -- a plain 4-read / 1-write kernel (tools/stream_ceiling.cu: 128-bit ld.global.nc, st.global.cs,
                  grid-stride loop), best of a few block / grid shapes;
  (b) staging  -- out = (x0 + x1) + (x2 + x3) through the library: the sweep kernel's staging, almost no compute;
  (c) c2       -- bench.py's 9-node expression without the reduction;
  (d) c2_hsum  -- the same with hsum() of its output, as bench.py runs it;
each in ms and in GB/s of algorithmic traffic (16 B read + 4 B written per element), plus the card name, power limit
and SM clock sampled during the run.  If (b) streams near (a) and (c) does not, C2 has compute that does not overlap
its loads; if (b) is itself near (c), the limit is the staging path.

    python tools/stream_probe.py [--elems N] [--reps R] [--json FILE]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import threading

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
BYTES_PER_ELEM = 20.0


class ClockSampler:
    """nvidia-smi SM clock sampled every 100 ms on a background thread (query only)."""

    def __init__(self):
        self.samples, self._stop, self._t = [], threading.Event(), None

    def _run(self):
        while not self._stop.wait(0.1):
            try:
                out = subprocess.run(["nvidia-smi", "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0],
                                      "--query-gpu=clocks.sm", "--format=csv,noheader,nounits"],
                                     capture_output=True, text=True, timeout=5).stdout.strip()
                self.samples.append(int(out.splitlines()[0]))
            except Exception:
                pass

    def __enter__(self):
        self._t = threading.Thread(target=self._run, daemon=True)
        self._t.start()
        return self

    def __exit__(self, *exc):
        self._stop.set()
        self._t.join()


def card_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=10).stdout.strip().splitlines()[0]
        name, plim, maxclk = (s.strip() for s in out.split(","))
        return {"name": name, "power_limit": plim, "max_sm_clock": maxclk}
    except Exception as e:
        return {"error": repr(e)}


def ceiling(n, reps, warmup):
    lib = ctypes.CDLL(os.path.join(ROOT, "tools", "libstream_ceiling.so"))
    lib.sc_ceiling.argtypes = [ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                               ctypes.POINTER(ctypes.c_float)]
    best = None
    shapes = []
    for block, ctas in ((256, 2), (256, 4), (256, 8), (512, 2), (512, 4), (1024, 2)):
        ms = ctypes.c_float()
        err = lib.sc_ceiling(n, block, ctas, warmup, reps, ctypes.byref(ms))
        if err != 0:
            raise SystemExit(f"stream_probe.py: ceiling kernel failed with CUDA error {err}")
        shapes.append({"block": block, "ctas_per_sm": ctas, "ms": ms.value})
        if best is None or ms.value < best["ms"]:
            best = shapes[-1]
    return best, shapes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--elems", type=int, default=1 << 26)
    ap.add_argument("--reps", type=int, default=30, help="timed launches per figure (the best one is reported)")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", metavar="FILE", help="also write the result as JSON to FILE")
    args = ap.parse_args()
    n = args.elems

    import numpy as np
    import enoki_b200 as ek
    from enoki_b200 import Float32, fmadd, exp, sin, sqrt, hsum
    L = ek.lib()
    if L.ek_device_count() == 0:
        raise SystemExit("stream_probe.py: no CUDA device visible")
    assert L.ek_init() == 0, L.ek_last_error()

    # the same synthetic inputs as bench.py's C2, generated on the device
    idx = ek.UInt32.arange(n)
    x = []
    for k in range(4):
        h = idx * np.uint32(2654435761 + 2 * k) + np.uint32(12345 * (k + 1))
        x.append(fmadd(Float32(h >> 8), Float32(8.0 / (1 << 24)), Float32(-4.0)))
    ek.cuda_eval(); ek.cuda_sync()
    del idx

    def staging():
        out = (x[0] + x[1]) + (x[2] + x[3])
        ek.cuda_eval()
        return out

    def c2(with_hsum):
        t = fmadd(x[0], x[1], x[2])
        u = exp(-(t * t))
        v = sin(fmadd(x[3], u, x[0]))
        out = fmadd(v, x[1], sqrt(abs(t)))
        del t, u, v
        s = hsum(out) if with_hsum else None
        ek.cuda_eval()
        return out, s

    def best_of(fn):
        for _ in range(args.warmup):
            fn()
        L.ek_set_timing(1)
        best, fast = None, 0
        for _ in range(args.reps):
            L.ek_stats_reset()
            keep = fn()
            st = ek.stats()
            assert int(st.sweep_launches) == 1, f"expected one sweep launch, got {int(st.sweep_launches)}"
            fast += int(st.fast_launches)
            best = st.last_kernel_ms if best is None else min(best, st.last_kernel_ms)
            del keep
        L.ek_set_timing(0)
        return best, "ek_fast_kernel" if fast == args.reps else "ek_sweep_kernel"

    def fig(ms, **kw):
        return dict(ms=ms, gbs=BYTES_PER_ELEM * n / (ms * 1e-3) / 1e9, **kw)

    with ClockSampler() as clk:
        cbest, shapes = ceiling(n, args.reps, args.warmup)
        res = {"elems": n, "bytes_per_elem": BYTES_PER_ELEM,
               "ceiling": fig(cbest["ms"], block=cbest["block"], ctas_per_sm=cbest["ctas_per_sm"], shapes=shapes)}
        for name, fn in (("staging", staging), ("c2", lambda: c2(False)), ("c2_hsum", lambda: c2(True))):
            ms, kern = best_of(fn)
            res[name] = fig(ms, kernel=kern)
    for name in ("staging", "c2", "c2_hsum"):
        res[name]["frac_of_ceiling"] = res["ceiling"]["ms"] / res[name]["ms"]
        res[name]["frac_of_datasheet"] = res[name]["gbs"] / 3350.0
    res["ceiling"]["frac_of_datasheet"] = res["ceiling"]["gbs"] / 3350.0
    res["card"] = card_info()
    res["sm_clock_mhz"] = {"min": min(clk.samples), "max": max(clk.samples), "samples": len(clk.samples)} if clk.samples else None
    res["datasheet_gbs"] = "3350 (H100 SXM, HBM3)"
    for name in ("ceiling", "staging", "c2", "c2_hsum"):
        r = res[name]
        print(f"{name:8s} {r['ms']:.4f} ms  {r['gbs']:7.1f} GB/s  {r.get('kernel', '')}")
    print(json.dumps(res))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
