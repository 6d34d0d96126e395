"""What an Enoki -> torch -> Enoki round trip costs, copying against aliasing.

For each size (Float32 elements), the median over --reps round trips of:
  copy   -- t = a.torch(); b = Float32.from_torch(t): two device-to-device copies, each bracketed by host
            synchronisations (torch_interop.py);
  alias  -- t = torch.from_dlpack(a); b = enoki_b200.from_dlpack(t): no copy, stream hand-offs only;
both timed with a host clock around the round trip followed by a synchronisation of both frameworks, so the alias
figure includes the same final wait.  Also the device time of one of the copies (CUDA events on the backend's stream,
averaged over --reps launches), and the card name and power limit read in the same run.

    python tools/interop_probe.py [--sizes 20,26] [--reps 50] [--json FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=10)
    if q.returncode != 0:
        raise SystemExit("interop_probe: nvidia-smi failed -- this script measures on the GPU only")
    name, power = (s.strip() for s in q.stdout.strip().splitlines()[0].split(","))
    return {"name": name, "power_limit": power}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="20,26", help="log2 of the element counts")
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--json")
    args = ap.parse_args()

    import numpy as np
    import torch
    import enoki_b200 as ek
    import enoki_b200.torch_interop  # noqa: F401  (.torch() / from_torch())
    if ek.device_count() == 0:
        raise SystemExit("interop_probe: no CUDA device")
    L = ek.lib()
    card = card_info()

    def sync():
        L.ek_sync()
        torch.cuda.synchronize()

    def copy_trip(a):
        return ek.Float32.from_torch(a.torch())

    def alias_trip(a):
        return ek.from_dlpack(torch.from_dlpack(a))

    results = []
    for lg in (int(s) for s in args.sizes.split(",")):
        n = 1 << lg
        a = ek.Float32.copy(np.linspace(-1, 1, n, dtype=np.float32))
        want = a.numpy()
        row = {"elems": n}
        for name, trip in (("copy", copy_trip), ("alias", alias_trip)):
            b = trip(a)                                   # warm-up, and the result is checked
            assert np.array_equal(b.numpy().view(np.uint32), want.view(np.uint32)), name
            del b
            sync()
            times = []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                b = trip(a)
                sync()
                times.append((time.perf_counter() - t0) * 1e3)
                del b
            row[name + "_ms"] = statistics.median(times)
        # device time of one copy of the buffer, as .torch() and from_torch() each issue it
        dst = L.ek_malloc(4 * n)
        L.ek_memcpy_device_async(dst, a.data(), 4 * n)
        L.ek_timer_start()
        for _ in range(args.reps):
            L.ek_memcpy_device_async(dst, a.data(), 4 * n)
        row["copy_kernel_ms"] = L.ek_timer_stop() / args.reps
        L.ek_free(dst)
        row["speedup"] = row["copy_ms"] / row["alias_ms"]
        results.append(row)
        del a
        sync()
    out = {"card": card, "reps": args.reps, "results": results}
    print(json.dumps(out))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
