"""Generate the golden vectors under tests/golden/ from the UNMODIFIED reference CPU path
(oracle/_ref/libenoki_ref.so = /root/reference headers + src/autodiff/autodiff.cpp built by
`make -C oracle ref`).  Run in the dev container (the reference does not travel to the GPU box);
the .npz files are committed.

    python tests/golden/make_golden.py
"""
import ctypes
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
R = ctypes.CDLL(os.path.join(ROOT, "oracle", "_ref", "libenoki_ref.so"))
P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
SZ = ctypes.c_size_t


def unary(name, x):
    out = np.zeros_like(x)
    assert R.ref_unary_f32(name.encode(), P(x), P(out), SZ(len(x))) == 0
    return out


def main():
    rng = np.random.default_rng(20260922)
    # --- C2: fused chain (SURVEY 8d) on 4099 elements
    n = 4099
    xs = [rng.uniform(-4, 4, n).astype(np.float32) for _ in range(4)]
    out = np.zeros(n, np.float32)
    R.ref_c2(*[P(x) for x in xs], P(out), SZ(n))
    np.savez_compressed(os.path.join(HERE, "c2.npz"), x0=xs[0], x1=xs[1], x2=xs[2], x3=xs[3], out=out)

    # --- C1: a*b + sin(c) (tests/dynamic.cpp path), linspace inputs of config #1 at reduced size
    n = 4096
    a = np.linspace(0, 1, n, dtype=np.float32); b = np.linspace(1, 2, n, dtype=np.float32); c = np.linspace(-3, 3, n, dtype=np.float32)
    out = np.zeros(n, np.float32)
    R.ref_c1(P(a), P(b), P(c), P(out), SZ(n))
    np.savez_compressed(os.path.join(HERE, "c1.npz"), a=a, b=b, c=c, out=out)

    # --- unary math on special + random values
    x = np.concatenate([np.array([0, -0.0, np.inf, -np.inf, np.nan, 1, -1, 1e-40, 88.5, -88.5, 8191.5, -8191.5], np.float32),
                        rng.uniform(-50, 50, 2000).astype(np.float32)])
    d = {"x": x}
    for name in ("sin", "cos", "exp", "log", "sqrt", "floor", "ceil", "round", "trunc", "tan", "asin", "acos", "atan",
                 "sinh", "cosh", "tanh", "erf"):
        d[name] = unary(name, x)
    np.savez_compressed(os.path.join(HERE, "unary.npz"), **d)

    # --- double-precision branches of sin/cos/exp/log
    x = np.concatenate([np.array([0, -0.0, np.inf, -np.inf, np.nan, 1, -1, 1e-310, 709.5, -709.5, 710, -710, 8191.5, -8191.5]),
                        rng.uniform(-700, 700, 1000), np.exp(rng.uniform(-700, 700, 1000))]).astype(np.float64)
    d = {"x": x}
    for name in ("sin", "cos", "exp", "log", "sqrt"):
        out = np.zeros_like(x)
        assert R.ref_unary_f64(name.encode(), P(x), P(out), SZ(len(x))) == 0
        d[name] = out
    np.savez_compressed(os.path.join(HERE, "unary_f64.npz"), **d)

    # --- C3 histogram: PCG32 samples -> erfinv -> 31 bins (tests/histogram.cpp:41-57), 2^16 samples
    n = 1 << 16
    u = np.zeros(n, np.float32)
    R.ref_pcg32_f32(ctypes.c_uint64(0), SZ(n), SZ(1), P(u))
    y = np.zeros(n, np.float32)
    R.ref_hist_samples(P(u), P(y), SZ(n))
    table = rng.uniform(0.5, 1.5, 31).astype(np.float32)
    idx = np.zeros(n, np.uint32); bins = np.zeros(31, np.uint32); hist = np.zeros(31, np.float32)
    R.ref_c3(P(y), SZ(n), P(table), P(idx), P(bins), P(hist))
    np.savez_compressed(os.path.join(HERE, "c3.npz"), u=u, y=y, table=table, idx=idx, bins=bins, hist=hist)

    # --- PCG32 raw draws
    m, draws = 257, 4
    pu = np.zeros(m * draws, np.uint32)
    R.ref_pcg32_u32(ctypes.c_uint64(0), SZ(m), SZ(draws), P(pu))
    np.savez_compressed(os.path.join(HERE, "pcg32.npz"), first=0, n=m, draws=draws, u32=pu)

    # --- tape: layered random graph (C4 shape, reduced): L levels x K nodes, width w, 2 in-edges per node
    for tag, (L, K, w) in {"small": (6, 8, 37), "wide": (4, 5, 1000)}.items():
        g = make_tape(rng, L, K, w)
        grads = np.zeros(len(g["want"]) * w, np.float32)
        rc = R.ref_tape_backward(len(g["node_size"]), P(g["node_size"]), len(g["src"]), P(g["src"]), P(g["dst"]),
                                 P(g["weights"]), P(g["woff"]), P(g["wsize"]), int(g["root"]), len(g["want"]), P(g["want"]),
                                 P(grads), 1)
        assert rc == 0
        np.savez_compressed(os.path.join(HERE, f"tape_{tag}.npz"), grads=grads, **g)

    # --- public-API autodiff expressions (tests/autodiff.cpp style)
    x = rng.uniform(0.2, 2.0, 513).astype(np.float32)
    d = {"x": x}
    for which in range(5):
        v = np.zeros_like(x); gr = np.zeros_like(x)
        assert R.ref_ad_expr(which, P(x), SZ(len(x)), P(v), P(gr)) == 0
        d[f"val{which}"] = v; d[f"grad{which}"] = gr
    np.savez_compressed(os.path.join(HERE, "ad_expr.npz"), **d)
    ref_math()
    ref_tape()
    ref_tape_sweep()
    convert()
    shim_plan()
    print("golden vectors written to", HERE)


# ek_type codes of the ten numeric types (include/enoki_b200.h)
CONVERT_TYPES = {"Int8": 1, "UInt8": 2, "Int16": 3, "UInt16": 4, "Int32": 5, "UInt32": 6, "Int64": 7, "UInt64": 8,
                 "Float32": 10, "Float64": 11}
CONVERT_DTYPES = {"Int8": np.int8, "UInt8": np.uint8, "Int16": np.int16, "UInt16": np.uint16, "Int32": np.int32,
                  "UInt32": np.uint32, "Int64": np.int64, "UInt64": np.uint64, "Float32": np.float32, "Float64": np.float64}


def convert_inputs(rng, tname):
    """One input vector per source type: the values where conversions change behaviour, then random ones."""
    dt = np.dtype(CONVERT_DTYPES[tname])
    if dt.kind == "f":
        fi = np.finfo(dt)
        v = [0.0, fi.smallest_subnormal, fi.smallest_normal - fi.smallest_subnormal, 0.5, 1.5, 2.5, 0.7, 1e19, 5e9, 3e9]
        for e in (7, 8, 15, 16, 31, 32, 53, 63, 64):
            b = dt.type(2.0 ** e)
            v += [np.nextafter(b, dt.type(0)), b, np.nextafter(b, dt.type(np.inf))]
        v = np.array(v, dt)
        v = np.concatenate([v, -v, np.array([np.inf, -np.inf, np.nan], dt)])
        emax = 128 if dt == np.float32 else 1024
        emin = -149 if dt == np.float32 else -1074
        mag = np.exp2(rng.uniform(emin, emax, 300)).astype(dt)
        mag = np.where(np.isinf(mag), fi.max, mag)
        sign = np.where(rng.random(300) < 0.5, -1, 1).astype(dt)
        return np.concatenate([v, mag * sign, (rng.uniform(-300, 300, 100)).astype(dt)]).astype(dt)
    info = np.iinfo(dt)
    w = 8 * dt.itemsize
    v = [info.min, info.max, -1, 0, 1, info.min + 1, info.max - 1]
    for e in (24, 53):
        v += [2 ** e - 1, 2 ** e + 1, -(2 ** e) - 1, -(2 ** e) + 1]
    if w == 64:
        v += [0x8000000000000001, 0x8000000000000000 + (1 << 40) + 1, 10 ** 19]
    wrap = lambda x: np.array([int(x) & ((1 << w) - 1)], "u%d" % dt.itemsize).view(dt)[0]
    v = np.array([wrap(x) for x in v if info.min <= x <= info.max or x >= 0 and info.min == 0 and x < 2 ** w], dt)
    full = rng.integers(info.min, info.max, 200, endpoint=True, dtype=dt)
    bits = rng.integers(1, w, 200)                       # magnitudes spread over every bit length
    logu = np.array([wrap(int(rng.integers(0, 1 << 62)) % (1 << int(b)) * (-1 if info.min < 0 and k & 1 else 1))
                     for k, b in enumerate(bits)], dt)
    return np.concatenate([v, full, logu])


def convert():
    """The reference's conversions between every ordered pair of the ten numeric types (converting constructor), and
    floor2int / ceil2int from Float32 and Float64 to the eight integer types (convert.npz).  x_<src> is the input of
    source type src; <src>_<dst>_<mode> the output, mode 0 = converting constructor, 1 = floor2int, 2 = ceil2int."""
    rng = np.random.default_rng(64)
    d = {}
    for src, sc in CONVERT_TYPES.items():
        x = np.ascontiguousarray(convert_inputs(rng, src))
        d[f"x_{src}"] = x
        for dst, dc in CONVERT_TYPES.items():
            modes = (0, 1, 2) if src.startswith("Float") and not dst.startswith("Float") else (0,)
            for mode in modes:
                out = np.zeros(len(x), CONVERT_DTYPES[dst])
                assert R.ref_convert(sc, dc, mode, P(x), P(out), SZ(len(x))) == 0, (src, dst, mode)
                d[f"{src}_{dst}_{mode}"] = out
    np.savez_compressed(os.path.join(HERE, "convert.npz"), **d)


# inputs of tests/test_cpu_oracle.py::test_oracle_vs_reference_math: (name, oracle selector, generator)
REF_MATH = [("sin", 0, lambda rng, n: rng.uniform(-8192, 8192, n)), ("cos", 1, lambda rng, n: rng.uniform(-8192, 8192, n)),
            ("exp", 2, lambda rng, n: rng.uniform(-100, 100, n)), ("log", 3, lambda rng, n: np.exp(rng.uniform(-80, 80, n))),
            ("sqrt", 4, lambda rng, n: rng.uniform(0, 1e10, n))]


def ref_math(n=1024):
    """The reference's float32 sin / cos / exp / log / sqrt on special values + random arguments (ref_math.npz)."""
    rng = np.random.default_rng(1)
    d = {}
    for name, _, gen in REF_MATH:
        x = gen(rng, n).astype(np.float32)
        x[:8] = [0, -0.0, np.inf, -np.inf, np.nan, 1, -1, 1e-40]
        d[f"x_{name}"] = x
        d[name] = unary(name, x)
    np.savez_compressed(os.path.join(HERE, "ref_math.npz"), **d)


def ref_tape(w=64):
    """The reference tape's backward() on a 7 x 12 layered graph of width w (ref_tape.npz)."""
    g = make_tape(np.random.default_rng(5), 7, 12, w)
    grads = np.zeros(len(g["want"]) * w, np.float32)
    assert R.ref_tape_backward(len(g["node_size"]), P(g["node_size"]), len(g["src"]), P(g["src"]), P(g["dst"]),
                               P(g["weights"]), P(g["woff"]), P(g["wsize"]), int(g["root"]), len(g["want"]), P(g["want"]),
                               P(grads), 1) == 0
    np.savez_compressed(os.path.join(HERE, "ref_tape.npz"), grads=grads, **g)


def ref_tape_sweep(n_graphs=48):
    """The reference tape's backward() and forward() from one seed on random general graphs (ref_tape_sweep.npz):
    tests/test_gpu_tape_graphs.random_graph with size-1 nodes joined to wide ones or not, with and without
    free_graph.  Every node's gradient is stored; an empty one reads as zeros."""
    import sys
    sys.path.insert(0, os.path.dirname(HERE))
    from test_gpu_tape_graphs import random_graph
    d = {}
    for k in range(n_graphs):
        rng = np.random.default_rng([21, k])
        forward, free_graph, mixed = k & 1, (k >> 1) & 1, (k >> 2) & 1
        g = random_graph(rng, 24, np.float32, mixed=bool(mixed), widths=(3, 4, 5, 17, 33, 67))
        n = len(g["node_size"])
        outs = np.bincount(g["src"].astype(np.int64), minlength=n + 1)
        root = int(np.argmax(outs)) if forward else n
        want = np.arange(1, n + 1, dtype=np.uint32)
        grads = np.zeros(int(g["node_size"].astype(np.int64).sum()), np.float32)
        fn = R.ref_tape_forward if forward else R.ref_tape_backward
        assert fn(n, P(g["node_size"]), len(g["src"]), P(g["src"]), P(g["dst"]), P(g["weights"]), P(g["woff"]),
                  P(g["wsize"]), root, n, P(want), P(grads), free_graph) == 0
        for key in ("node_size", "src", "dst", "weights", "woff", "wsize"):
            d[f"{k}_{key}"] = g[key]
        d[f"{k}_mode"] = np.array([forward, free_graph, root], np.uint32)
        d[f"{k}_grads"] = grads
    np.savez_compressed(os.path.join(HERE, "ref_tape_sweep.npz"), n_graphs=n_graphs, **d)


def shim_plan():
    """What tests/cpp/shim_plan (user C++ code over include/enoki/cuda.h and the reference's headers, built by
    `make -C tests/cpp shim_plan`) prints: the planner's listing of the programs it records (shim_plan.txt)."""
    import subprocess
    out = subprocess.run([os.path.join(ROOT, "tests", "cpp", "shim_plan")], capture_output=True, text=True, check=True).stdout
    with open(os.path.join(HERE, "shim_plan.txt"), "w") as f:
        f.write(out)


def make_tape(rng, L, K, w, zero_frac=0.01):
    """SURVEY 8d C4 generator: L levels x K nodes of width w; every non-leaf node has 2 in-edges
    to random nodes of the previous level; weights U(0.5,1.5) with a few exact zeros; loss = size-1
    node with a weight-1 edge from every node of the last level."""
    node_size, src, dst, woff, wsize, ws = [], [], [], [], [], []
    off = 0
    for lvl in range(L):
        for k in range(K):
            node_size.append(w)
            nid = lvl * K + k + 1
            if lvl > 0:
                picks = rng.choice(K, 2, replace=False)
                for p in sorted(picks):
                    src.append((lvl - 1) * K + int(p) + 1); dst.append(nid)
                    wt = rng.uniform(0.5, 1.5, w).astype(np.float32)
                    wt[rng.uniform(0, 1, w) < zero_frac] = 0.0
                    ws.append(wt); woff.append(off); wsize.append(w); off += w
    node_size.append(1)
    loss = L * K + 1
    for k in range(K):
        src.append((L - 1) * K + k + 1); dst.append(loss)
        ws.append(np.ones(1, np.float32)); woff.append(off); wsize.append(1); off += 1
    return dict(node_size=np.array(node_size, np.uint32), src=np.array(src, np.uint32), dst=np.array(dst, np.uint32),
                weights=np.concatenate(ws), woff=np.array(woff, np.uint64), wsize=np.array(wsize, np.uint32),
                root=np.uint32(loss), want=np.arange(1, K + 1, dtype=np.uint32))


if __name__ == "__main__":
    main()
