"""General tape graphs on the GPU against the oracle's or_tape_sweep_f32 / or_tape_sweep_f64.

The graphs are driven through the C ABI (ek_tape_*) in Float32 and Float64: random DAGs whose nodes have
mixed widths, edges that skip levels, duplicated edges, and every operand kind of the adjoint kernel (full,
evaluated size-1, literal, unevaluated and misaligned weights).  They run in backward and forward mode with
one or several seeds and with retained graphs.  Special edges, graph simplification and the local partials
of the Python FloatD ops are tested here too.

Comparisons are bit for bit (NaN == NaN).  The evaluator's hsum folds in a different order from the
reference's 8-lane packets, so graphs where a size-1 node sums a wide product (backward: size-1 sources of
wide edges; forward: size-1 targets of wide sources) carry small integer values, checked beforehand to keep
every partial sum exact.  Graph simplification is off except where a test turns it on.
"""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
F32, F64 = 10, 11
NP = {F32: np.float32, F64: np.float64}
WIDTHS = (3, 4, 5, 2047, 2048, 2049, 4099, (1 << 17) + 1)
KINDS = ("full", "scalar", "imm", "expr", "misaligned")


def _P(a):
    return a.ctypes.data_as(ctypes.c_void_p)


# ---- graph description (the oracle's format) ---------------------------------------------------------------
def random_graph(rng, n_nodes, dtype, mixed, widths=WIDTHS, ints=False, n_hubs=3):
    """Random DAG; node ids are creation order.  Every non-leaf node picks its sources among earlier nodes of
    the same width (with `mixed`, size-1 nodes also connect to wide ones and back): the first `n_hubs` of them
    feed most nodes (up to ~40 out-edges), the others are drawn from all earlier nodes, so edges skip levels.
    About one node in four repeats an edge, which the tape merges by adding the weights.  Weights are one of
    KINDS; float graphs put exact zeros and inf / NaN at a few shared element positions."""
    ws_pick = list(rng.choice(widths, 2, replace=False))
    sizes = [1 if (mixed and rng.random() < 0.25) or (not mixed and rng.random() < 0.1) else int(rng.choice(ws_pick))
             for _ in range(n_nodes)]
    n_leaves = max(3, n_nodes // 5)

    def compatible(a, b):
        return a == b or (mixed and (a == 1 or b == 1))

    src, dst, kinds, warrs = [], [], [], []
    hot = rng.integers(0, 1 << 30, 8)
    for i in range(n_leaves + 1, n_nodes + 1):
        si = sizes[i - 1]
        cands = [j for j in range(1, i) if compatible(sizes[j - 1], si)]
        if not cands:
            continue
        picks = [j for j in cands[:n_hubs] if rng.random() < 0.9]
        others = [j for j in cands if j not in picks]
        if others:
            picks += [int(j) for j in rng.choice(others, min(len(others), int(rng.integers(1, 4))), replace=False)]
        if not picks:
            picks = [cands[-1]]
        if rng.random() < 0.25:
            picks.append(picks[int(rng.integers(0, len(picks)))])          # duplicate edge
        wide_kind = {}
        for j in picks:
            sj = sizes[j - 1]
            wide = max(si, sj)
            # a repeated edge keeps the first weight's size: the reference adds the weights in place, which
            # only works for equal sizes
            choices = KINDS if j not in wide_kind else (("full", "expr", "misaligned") if wide_kind[j] else ("scalar", "imm"))
            kind = "scalar" if wide == 1 else str(rng.choice(choices))
            wide_kind.setdefault(j, kind in ("full", "expr", "misaligned"))
            n = wide if kind in ("full", "expr", "misaligned") else 1
            if ints:
                w = rng.choice(np.array([-1, 0, 1, 1, 2], dtype), n)
            else:
                w = rng.uniform(-1.5, 1.5, n).astype(dtype)
                w[rng.random(n) < 0.05] = 0
                if n > 1:
                    pos = hot % n
                    r = rng.random()
                    if r < 0.25:
                        w[pos[:3]] = np.array([np.inf, -np.inf, np.nan], dtype)
                    elif r < 0.6:
                        w[pos] = 0
            src.append(j); dst.append(i); kinds.append(kind); warrs.append(w)
    return make_graph(sizes, src, dst, warrs, kinds, dtype)


def make_graph(sizes, src, dst, warrs, kinds, dtype):
    woff = np.cumsum([0] + [len(w) for w in warrs[:-1]]).astype(np.uint64) if warrs else np.zeros(0, np.uint64)
    return dict(node_size=np.array(sizes, np.uint32), src=np.array(src, np.uint32), dst=np.array(dst, np.uint32),
                weights=np.concatenate(warrs).astype(dtype) if warrs else np.zeros(0, dtype), woff=woff,
                wsize=np.array([len(w) for w in warrs], np.uint32), kinds=list(kinds))


def reach(g, start, forward):
    """Nodes the set_gradient DFS schedules from `start`."""
    adj = {}
    for s, d in zip(g["src"].tolist(), g["dst"].tolist()):
        adj.setdefault(s if forward else d, []).append(d if forward else s)
    seen, stack = set(), [start]
    while stack:
        k = stack.pop()
        if k not in seen:
            seen.add(k)
            stack += adj.get(k, [])
    return seen


def best_start(g, forward):
    """The node whose sweep reaches the most elements."""
    sizes = g["node_size"].astype(np.int64)
    return max(range(1, len(sizes) + 1), key=lambda k: (sum(sizes[j - 1] for j in reach(g, k, forward)), k))


def oracle_sweep(oracle, g, seeds, forward, free_graph=True, want=None):
    """seeds: [(node id, values of size 1 or the node's size)] in set_gradient order; want: node ids (default all).
    Returns the concatenated gradients (empty ones read as zeros) and the return code."""
    dt = g["weights"].dtype
    fn = oracle.or_tape_sweep_f32 if dt == np.float32 else oracle.or_tape_sweep_f64
    want = np.arange(1, len(g["node_size"]) + 1, dtype=np.uint32) if want is None else np.array(want, np.uint32)
    seed_ids = np.array([s for s, _ in seeds], np.uint32)
    vals = [np.atleast_1d(np.asarray(v, dt)) for _, v in seeds]
    seed_vals = np.concatenate(vals).astype(dt)
    seed_off = np.cumsum([0] + [len(v) for v in vals[:-1]]).astype(np.uint64)
    seed_size = np.array([len(v) for v in vals], np.uint32)
    out = np.zeros(int(g["node_size"][want - 1].astype(np.int64).sum()), dt)
    rc = fn(int(forward), int(free_graph), len(g["node_size"]), _P(g["node_size"]), len(g["src"]), _P(g["src"]),
            _P(g["dst"]), _P(g["weights"]), _P(g["woff"]), _P(g["wsize"]), len(seeds), _P(seed_ids), _P(seed_vals),
            _P(seed_off), _P(seed_size), len(want), _P(want), _P(out))
    return out, rc


def exact_bound(oracle, g, seeds, forward):
    """Bound on the magnitude of every partial sum: the same sweep in float64 on max(|weight|, 1) and |seed|.
    Every scheduled node has a path to a node whose gradient stays readable, and weights >= 1 make that node's
    value at least as large as any sum along the path."""
    ga = dict(g, weights=np.maximum(np.abs(g["weights"]), 1).astype(np.float64))
    out, rc = oracle_sweep(oracle, ga, [(s, np.abs(np.asarray(v, np.float64))) for s, v, *_ in seeds], forward)
    assert rc == 0
    return float(out.max(initial=0))


def int_graph(oracle, rng, n_nodes, dtype, seeds_of, forward, widths=WIDTHS[:7], mixed=True):
    """An integer-valued graph on which every partial sum is exact in `dtype`, with its seeds."""
    limit = 2.0 ** (24 if dtype == np.float32 else 53)
    for _ in range(50):
        g = random_graph(rng, n_nodes, dtype, mixed=mixed, widths=widths, ints=True)
        seeds = seeds_of(g)
        if exact_bound(oracle, g, seeds, forward) < limit:
            return g, seeds
    raise AssertionError("no exactly representable integer graph found")


def safe_mul(a, b):
    return np.where((a == 0) | (b == 0), a.dtype.type(0), a * b)


def safe_fmadd(a, b, c):
    """Exact for the integer data it is used on (no rounding between the product and the sum)."""
    return np.where((a == 0) | (b == 0), c, c + a * b)


def assert_same(got, want, what=""):
    assert got.shape == want.shape, (what, got.shape, want.shape)
    u = np.uint32 if got.dtype == np.float32 else np.uint64
    same = (got.view(u) == want.view(u)) | (np.isnan(got) & np.isnan(want))
    bad = np.flatnonzero(~same)
    assert bad.size == 0, f"{what}: {bad.size}/{same.size} differ, first at {bad[:5]}: got {got[bad[:5]]}, want {want[bad[:5]]}"


# ---- the same graph on the GPU tape ------------------------------------------------------------------------
class GpuTape:
    """Builds a graph description on the GPU tape of type `t` and owns what it allocated."""

    def __init__(self, ek, t, g):
        self.ek, self.t, self.g = ek, t, g
        self.L = ek.lib()
        self.cls = ek.Float32 if t == F32 else ek.Float64
        self.keep, self.bases = [], []
        n = len(g["node_size"])
        self.ids = [0] * (n + 1)
        e, E = 0, len(g["dst"])
        for i in range(1, n + 1):
            size = int(g["node_size"][i - 1])
            if e < E and g["dst"][e] == i:
                self.ids[i] = self.L.ek_tape_append_node(t, size, b"n")
                while e < E and g["dst"][e] == i:
                    off, ws = int(g["woff"][e]), int(g["wsize"][e])
                    w = self.var(g["weights"][off:off + ws], g["kinds"][e])
                    assert self.L.ek_tape_append_edge(t, self.ids[int(g["src"][e])], self.ids[i], w.index) == 0, \
                        self.L.ek_last_error()
                    e += 1
            else:
                self.ids[i] = self.L.ek_tape_append_leaf(t, size)

    def var(self, a, kind):
        """An evaluator variable holding `a` as the given operand kind."""
        a = np.ascontiguousarray(a, NP[self.t])
        if kind == "imm":
            v = self.cls(a[0].item())
        elif kind == "scalar":
            v = self.cls.copy(a[:1])
        elif kind == "full":
            v = self.cls.copy(a)
        elif kind == "expr":                             # unevaluated: backward() must evaluate it first
            v = self.cls.copy(a) * 1.0
        elif kind == "misaligned":                       # one element off 16-byte alignment: scalar loads
            es = a.itemsize
            p = self.L.ek_malloc((a.size + 1) * es)
            self.L.ek_memcpy_to_device(p + es, a.ctypes.data, a.nbytes)
            self.bases.append(p)
            v = self.cls.map(p + es, a.size)
        else:
            raise ValueError(kind)
        self.keep.append(v)
        return v

    def seed(self, node, values, kind, backward):
        v = self.var(np.atleast_1d(values), kind)
        assert self.L.ek_tape_set_gradient(self.t, self.ids[node], v.index, int(backward)) == 0, self.L.ek_last_error()

    def run(self, backward, free_graph):
        f = self.L.ek_tape_backward_static if backward else self.L.ek_tape_forward_static
        assert f(self.t, int(free_graph)) == 0, self.L.ek_last_error().decode()

    def handle(self, node):
        return self.L.ek_tape_gradient(self.t, self.ids[node])

    def grads(self, want=None):
        want = range(1, len(self.g["node_size"]) + 1) if want is None else want
        outs = []
        for k in want:
            sz = int(self.g["node_size"][k - 1])
            h = self.handle(k)
            if h == 0:
                outs.append(np.zeros(sz, NP[self.t]))
                continue
            self.L.ek_inc_ref_ext(h)
            a = self.cls.from_index(h).numpy()
            outs.append(np.broadcast_to(a, (sz,)).copy() if a.size == 1 else a)
        return np.concatenate(outs)

    def release(self):
        for i in self.ids[1:]:
            self.L.ek_tape_dec_ref_ext(self.t, i)
        self.keep.clear()
        self.L.ek_sync()
        for p in self.bases:
            self.L.ek_free(p)
        self.bases.clear()
        assert self.L.ek_tape_node_count(self.t) == 0


@pytest.fixture()
def tape(gpu):
    L = gpu.lib()
    for t in (F32, F64):
        L.ek_tape_set_graph_simplification(t, 0)
    yield gpu
    for t in (F32, F64):
        L.ek_tape_clear(t)                               # whatever a failed test left behind
        L.ek_tape_set_graph_simplification(t, 1)


def sweep_and_compare(ek, oracle, t, g, seeds, backward, free_graph=True, what=""):
    """seeds: [(node, values, kind)]; runs the GPU tape and the oracle and compares every node's gradient."""
    want, rc = oracle_sweep(oracle, g, [(s, v) for s, v, _ in seeds], not backward, free_graph)
    assert rc == 0
    gt = GpuTape(ek, t, g)
    for s, v, kind in seeds:
        gt.seed(s, v, kind, backward)
    gt.run(backward, free_graph)
    assert_same(gt.grads(), want, what)
    gt.release()


def seeds_for(g, rng, how, backward, dtype):
    """Seed list [(node, values, kind)] for a graph: `how` picks one of the seedings the tests cover."""
    n = len(g["node_size"])
    sizes = g["node_size"]
    start = best_start(g, not backward)
    size = int(sizes[start - 1])
    vals = lambda k: (rng.choice([-3, -2, -1, 1, 2, 3], k) if dtype is None else rng.uniform(-2, 2, k)).astype(dtype or np.float64)
    if how == "one":
        return [(start, 1.0, "imm")]
    if how == "wide":
        return [(start, vals(size), "full")]
    if how == "scalar":
        return [(start, vals(1), "imm")]
    if how == "misaligned":
        return [(start, vals(size), "misaligned" if size > 1 else "scalar")]
    if how == "two":                                  # the second seed is reached from the first and keeps its value
        inner = sorted(reach(g, start, not backward) - {start})
        other = inner[len(inner) // 2] if inner else start
        osz = int(sizes[other - 1])
        return [(other, vals(osz), "full" if osz > 1 else "scalar"), (start, vals(size), "full" if size > 1 else "scalar")]
    raise ValueError(how)


# ---- random DAGs -------------------------------------------------------------------------------------------
SEEDINGS = ("one", "wide", "scalar", "two", "misaligned")


@pytest.mark.parametrize("t", [F32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("backward", [True, False], ids=["backward", "forward"])
@pytest.mark.parametrize("how", SEEDINGS)
def test_random_dag_float(tape, oracle, t, backward, how):
    """Random float data, bit for bit: wide nodes and size-1 nodes that only meet each other."""
    dt = NP[t]
    rng = np.random.default_rng([t, backward, SEEDINGS.index(how)])
    g = random_graph(rng, 64, dt, mixed=False)
    seeds = seeds_for(g, rng, how, backward, dt)
    sweep_and_compare(tape, oracle, t, g, [(s, np.asarray(v, dt), k) for s, v, k in seeds], backward,
                      what=f"{how} seed")


@pytest.mark.parametrize("t", [F32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("backward", [True, False], ids=["backward", "forward"])
@pytest.mark.parametrize("how", SEEDINGS)
def test_random_dag_mixed_sizes(tape, oracle, t, backward, how):
    """Size-1 nodes connected to wide ones (hsum and broadcast on the generic path), integer-valued so that
    the evaluator's hsum order cannot change a bit."""
    dt = NP[t]
    rng = np.random.default_rng([7, t, backward, SEEDINGS.index(how)])
    g, seeds = int_graph(oracle, rng, 40, dt, lambda g: [(s, np.asarray(v, dt), k) for s, v, k in
                                                          seeds_for(g, rng, how, backward, None)], not backward)
    sweep_and_compare(tape, oracle, t, g, [(s, np.asarray(v, dt), k) for s, v, k in seeds], backward,
                      what=f"{how} seed")


# ---- retained graphs ---------------------------------------------------------------------------------------
def _c4_graph(rng, dtype):
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
    from make_golden import make_tape
    g = make_tape(rng, 6, 24, 4099)
    g = dict(g, weights=g["weights"].astype(dtype), kinds=["full" if ws > 1 else "imm" for ws in g["wsize"]])
    return g, int(g["root"])


@pytest.mark.parametrize("t", [F32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("shape", ["c4", "random"])
def test_backward_retained_graph(tape, oracle, t, shape):
    """backward(free_graph=False) three times, then backward(True): every pass computes the same sweep, a
    retained pass leaves readable only the gradients of nodes without out-edges (autodiff.cpp:895-897), and the
    final pass frees the whole graph."""
    dt = NP[t]
    rng = np.random.default_rng([11, t])
    if shape == "c4":
        g, root = _c4_graph(rng, dt)
    else:
        g = random_graph(rng, 64, dt, mixed=False)
        root = best_start(g, False)
    L = tape.lib()
    keep_r, rc = oracle_sweep(oracle, g, [(root, 1.0)], False, free_graph=False)
    final, rc2 = oracle_sweep(oracle, g, [(root, 1.0)], False, free_graph=True)
    assert rc == 0 and rc2 == 0
    gt = GpuTape(tape, t, g)
    has_out, has_in = set(g["src"].tolist()), set(g["dst"].tolist())
    sched = reach(g, root, False)
    # readable after a retained pass: scheduled nodes without out-edges (the root) and unscheduled leaves
    readable = [k for k in range(1, len(g["node_size"]) + 1) if (k not in has_out if k in sched else k not in has_in)]
    for _ in range(3):
        assert L.ek_tape_backward(t, gt.ids[root], 0) == 0, L.ek_last_error()
        assert [k for k in range(1, len(g["node_size"]) + 1) if gt.handle(k) != 0] == readable
        assert_same(gt.grads(), keep_r, "retained pass")
    n_before = L.ek_tape_node_count(t)
    assert L.ek_tape_backward(t, gt.ids[root], 1) == 0, L.ek_last_error()
    assert_same(gt.grads(), final, "final pass")
    assert L.ek_tape_node_count(t) == n_before
    gt.release()


@pytest.mark.parametrize("t", [F32, F64], ids=["f32", "f64"])
def test_forward_retained_graph(tape, oracle, t):
    """forward(x, False), read every gradient, then forward(y): both against the oracle.  Nodes the second pass
    does not reach keep what the first pass left."""
    dt = NP[t]
    rng = np.random.default_rng([12, t])
    g = random_graph(rng, 48, dt, mixed=False)
    leaves = [k for k in range(1, len(g["node_size"]) + 1) if k not in set(int(d) for d in g["dst"])]
    outs = np.bincount(g["src"].astype(np.int64), minlength=len(g["node_size"]) + 1)
    x, y = sorted(leaves, key=lambda k: -outs[k])[:2]
    first, rc = oracle_sweep(oracle, g, [(x, 1.0)], True, free_graph=False)
    second, rc2 = oracle_sweep(oracle, g, [(y, 1.0)], True, free_graph=True)
    assert rc == 0 and rc2 == 0
    ry = reach(g, y, True)
    sel = np.concatenate([np.full(int(s), k in ry) for k, s in enumerate(g["node_size"], 1)])
    second = np.where(sel, second, first)
    L = tape.lib()
    gt = GpuTape(tape, t, g)
    assert L.ek_tape_forward(t, gt.ids[x], 0) == 0, L.ek_last_error()
    assert_same(gt.grads(), first, "forward(x, False)")
    assert L.ek_tape_forward(t, gt.ids[y], 1) == 0, L.ek_last_error()
    assert_same(gt.grads(), second, "forward(y)")
    gt.release()


# ---- levels ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t", [F32, F64], ids=["f32", "f64"])
def test_level_with_many_mixed_jobs(tape, oracle, t):
    """One level of 2 100 sources of mixed widths: more chunks than the grid has CTAs, so CTAs stride over
    chunks and the chunk search crosses many job boundaries."""
    dt = NP[t]
    rng = np.random.default_rng([13, t])
    widths = (3, 4, 5, 2047, 2048, 2049, 4099)
    n_leaves = 2100
    sizes = [widths[i % len(widths)] for i in range(n_leaves)] + [w for w in widths for _ in range(2)] + [1]
    tid = {w: (n_leaves + 1 + 2 * k, n_leaves + 2 + 2 * k) for k, w in enumerate(widths)}
    edges = []
    for i in range(1, n_leaves + 1):
        w = sizes[i - 1]
        for tg in (tid[w] if rng.random() < 0.5 else (tid[w][int(rng.integers(0, 2))],)):
            edges.append((i, tg, str(rng.choice(("full", "scalar", "imm", "misaligned")))))
    root = len(sizes)
    edges += [(k, root, "imm") for k in range(n_leaves + 1, root)]
    edges.sort(key=lambda e: e[1])
    warrs = []
    for s, d, kind in edges:
        n = sizes[s - 1] if kind in ("full", "misaligned") else 1
        warrs.append(rng.uniform(-1.5, 1.5, n).astype(dt))
    g = make_graph(sizes, [e[0] for e in edges], [e[1] for e in edges], warrs, [e[2] for e in edges], dt)
    sweep_and_compare(tape, oracle, t, g, [(root, 1.0, "imm")], True)


@pytest.mark.parametrize("t", [F32, F64], ids=["f32", "f64"])
def test_level_mixing_generic_and_kernel_sources(tape, t):
    """One level holds a kernel source (A), a size-1 source of wide edges (B, hsum) and the source of a reverse
    edge that also has an ordinary edge (C); all three feed the same targets R and T."""
    dt = NP[t]
    rng = np.random.default_rng([14, t])
    n = 4099
    L = tape.lib()
    cls = tape.Float32 if t == F32 else tape.Float64
    iv = lambda k: rng.integers(-3, 4, k).astype(dt)
    w = {k: iv(n) for k in ("AR", "BR", "RT", "CT", "AT", "BT")}
    g = iv(n)
    C = L.ek_tape_append_leaf(t, n)
    A = L.ek_tape_append_leaf(t, n)
    B = L.ek_tape_append_leaf(t, 1)
    R = L.ek_tape_append_reverse(t, C)
    keep = {k: cls.copy(v) for k, v in w.items()}
    assert L.ek_tape_append_edge(t, A, R, keep["AR"].index) == 0
    assert L.ek_tape_append_edge(t, B, R, keep["BR"].index) == 0
    T = L.ek_tape_append_node(t, n, b"T")
    for s, k in ((R, "RT"), (C, "CT"), (A, "AT"), (B, "BT")):
        assert L.ek_tape_append_edge(t, s, T, keep[k].index) == 0
    seed = cls.copy(g)
    assert L.ek_tape_set_gradient(t, T, seed.index, 1) == 0
    assert L.ek_tape_backward_static(t, 1) == 0, L.ek_last_error()

    def grad(i):
        h = L.ek_tape_gradient(t, i)
        L.ek_inc_ref_ext(h)
        return cls.from_index(h).numpy()

    # out-edges in descending target id (T before R); integer data, so only the zero guards shape the bits
    gR = safe_mul(w["RT"], g)
    assert_same(grad(A), safe_fmadd(w["AR"], gR, safe_mul(w["AT"], g)), "A")
    assert_same(grad(B), np.array([np.sum(safe_mul(w["BT"], g)) + np.sum(safe_mul(w["BR"], gR))], dt), "B")
    assert_same(grad(C), safe_mul(w["CT"], g) + gR[::-1], "C")
    for i in (C, A, B, R, T):
        L.ek_tape_dec_ref_ext(t, i)
    assert L.ek_tape_node_count(t) == 0


@pytest.mark.parametrize("t", [F32, F64], ids=["f32", "f64"])
def test_forward_broadcasts_size1_gradients(tape, oracle, t):
    """Forward mode: a size-1 source feeds a wide node through a size-1 weight, so the wide node's gradient must
    be broadcast (autodiff.cpp:955-965) before it is summed into a size-1 target: grad(z) = hsum(2 * 3) over n."""
    dt = NP[t]
    n = 2049
    g = make_graph([1, n, 1], [1, 2], [2, 3], [np.array([3], dt), np.array([2], dt)], ["imm", "imm"], dt)
    sweep_and_compare(tape, oracle, t, g, [(1, 1.0, "imm")], False)
    want, _ = oracle_sweep(oracle, g, [(1, 1.0)], True, want=[3])
    assert want[0] == 6 * n


# ---- special edges -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("t", [F32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("masked", [False, True], ids=["all", "masked"])
def test_scatter_into_leaf_then_backward(tape, t, masked):
    """scatter(x) into a leaf, then set_gradient + backward_static with nothing evaluated in between: the
    leaf's gradient is 0 at the overwritten slots and g elsewhere (masked-out lanes write nothing, so their
    slots keep g), and x receives gather(g) where its lanes were written."""
    ek = tape
    L = ek.lib()
    dt = NP[t]
    cls = ek.Float32 if t == F32 else ek.Float64
    rng = np.random.default_rng([15, t, masked])
    n, m = 10_007, 3_001
    idx = rng.permutation(n)[:m].astype(np.uint32)
    mask = rng.random(m) < 0.7 if masked else np.ones(m, bool)
    g = rng.uniform(-2, 2, n).astype(dt)
    tgt = L.ek_tape_append_leaf(t, n)
    x = L.ek_tape_append_leaf(t, m)
    off, msk = ek.UInt32.copy(idx), ek.Mask.copy(mask)
    L.ek_tape_inc_ref_ext(t, tgt)                      # append_scatter drops the operand's reference
    cur = ctypes.c_uint32(tgt)
    assert L.ek_tape_set_scatter_gather_operand(t, ctypes.byref(cur), n, 0) == 0
    assert L.ek_tape_append_scatter(t, x, off.index, msk.index, 0) == 0, L.ek_last_error()
    assert L.ek_tape_set_scatter_gather_operand(t, None, 0, 0) == 0
    out = cur.value
    assert out != tgt
    seed = cls.copy(g)
    assert L.ek_tape_set_gradient(t, out, seed.index, 1) == 0
    assert L.ek_tape_backward_static(t, 1) == 0, L.ek_last_error()

    def grad(i):
        h = L.ek_tape_gradient(t, i)
        L.ek_inc_ref_ext(h)
        a = cls.from_index(h).numpy()
        return a
    want_t = g.copy()
    want_t[idx[mask]] = 0
    assert_same(grad(tgt), want_t, "scatter target")
    assert_same(grad(x), np.where(mask, g[idx], 0).astype(dt), "scattered source")
    L.ek_tape_dec_ref_ext(t, tgt)
    for i in (tgt, x, out):
        L.ek_tape_dec_ref_ext(t, i)
    assert L.ek_tape_node_count(t) == 0


@pytest.mark.parametrize("t", [F32, F64], ids=["f32", "f64"])
def test_forward_through_psum_and_reverse(tape, t):
    """Forward mode through psum and reverse edges (autodiff.cpp:430-440, 480-490), 3 * 524 288 + 5 elements of
    integer data (every prefix sum exact), and on into an ordinary edge that adds both."""
    ek = tape
    L = ek.lib()
    dt = NP[t]
    cls = ek.Float32 if t == F32 else ek.Float64
    n = 3 * 524_288 + 5
    rng = np.random.default_rng([16, t])
    g = rng.integers(-3, 4, n).astype(dt)
    w = rng.integers(-2, 3, n).astype(dt)
    x = L.ek_tape_append_leaf(t, n)
    p = L.ek_tape_append_psum(t, x)
    r = L.ek_tape_append_reverse(t, x)
    wv, one = cls.copy(w), cls(1.0)
    z = L.ek_tape_append_node(t, n, b"z")
    assert L.ek_tape_append_edge(t, p, z, wv.index) == 0
    assert L.ek_tape_append_edge(t, r, z, one.index) == 0
    seed = cls.copy(g)
    assert L.ek_tape_set_gradient(t, x, seed.index, 0) == 0
    assert L.ek_tape_forward_static(t, 1) == 0, L.ek_last_error()
    h = L.ek_tape_gradient(t, z)
    L.ek_inc_ref_ext(h)
    ps = np.cumsum(g.astype(np.float64)).astype(dt)
    want = np.where(w == 0, 0, w * ps).astype(dt) + g[::-1]
    assert_same(cls.from_index(h).numpy(), want.astype(dt), "forward psum / reverse")
    for i in (x, p, r, z):
        L.ek_tape_dec_ref_ext(t, i)
    assert L.ek_tape_node_count(t) == 0


# ---- simplification ----------------------------------------------------------------------------------------
def _parallel_collapses(g):
    """(a, n, o) triples where collapsing n turns a -> n -> o into an edge parallel to an existing a -> o."""
    E = set(zip(g["src"].tolist(), g["dst"].tolist()))
    ins, outs = {}, {}
    for s, d in E:
        outs.setdefault(s, set()).add(d)
        ins.setdefault(d, set()).add(s)
    return [(a, k, o) for k in ins if k in outs for a in ins[k] for o in outs[k] if (a, o) in E]


@pytest.mark.parametrize("t", [F32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("k", range(3))
def test_simplification_keeps_gradients(tape, oracle, t, k):
    """Integer-valued random DAGs: backward after ek_tape_simplify is bit-identical to the oracle on the
    unsimplified graph (every product and sum is exact), including collapses whose new edge runs parallel to an
    existing one.  Size-1 nodes only meet size-1 nodes here: collapsing a wide node between two size-1 nodes
    leaves a wide weight on a size-1 -> size-1 edge, which this test does not cover."""
    dt = NP[t]
    rng = np.random.default_rng([17, t, k])
    widths = (5, 2049, 4099)

    def seeds_of(g):
        return [(best_start(g, False), np.array([1.0], dt))]
    for _ in range(20):
        g, seeds = int_graph(oracle, rng, 30, dt, seeds_of, False, widths=widths, mixed=False)
        if _parallel_collapses(g):
            break
    assert _parallel_collapses(g)
    root = seeds[0][0]
    want, rc = oracle_sweep(oracle, g, seeds, False)
    assert rc == 0
    L = tape.lib()
    gt = GpuTape(tape, t, g)
    srcs, dsts = set(g["src"].tolist()), set(g["dst"].tolist())
    n = len(g["node_size"])
    interior = [i for i in range(1, n + 1) if i in srcs and i in dsts and i != root]
    for i in interior:                                  # interior nodes are referenced by the graph only
        L.ek_tape_dec_ref_ext(t, gt.ids[i])
    n_before = L.ek_tape_node_count(t)
    assert L.ek_tape_simplify(t) == 0
    assert L.ek_tape_node_count(t) < n_before
    assert L.ek_tape_backward(t, gt.ids[root], 1) == 0, L.ek_last_error()
    kept = [i for i in range(1, n + 1) if i not in interior]
    sel = np.concatenate([np.full(int(s), i in kept) for i, s in enumerate(g["node_size"], 1)])
    assert_same(gt.grads(kept), want[sel], "simplified")
    for i in kept:
        L.ek_tape_dec_ref_ext(t, gt.ids[i])
    gt.keep.clear()
    gt.L.ek_sync()
    for p in gt.bases:
        L.ek_free(p)
    assert L.ek_tape_node_count(t) == 0


# ---- FloatD partials ---------------------------------------------------------------------------------------
def _inputs(rng):
    """Edge values for the partials: +-0, denormals, large sin/cos arguments, values near exp overflow."""
    special = np.array([0.0, -0.0, 1e-40, -1e-40, 1.4e-45, 1e-38, 8191.5, -8000.25, 1e5, 88.3, 88.37, 88.8,
                        -87.5, -103.0, 1.0, -1.0, 3.0e38, np.inf, -np.inf, np.nan], np.float32)
    nan_neg = np.array([0xffc00000], np.uint32).view(np.float32)
    return np.concatenate([special, nan_neg, rng.uniform(-10, 10, 4096).astype(np.float32)])


def _div_pairs(rng):
    """a / b pairs where rcp(b)^2 overflows (or underflows), so (-a * rb) * rb and -a * (rb * rb) differ."""
    b = np.array([1e-20, -1e-25, 1e-30, 3e19, 1e25, 2.0, -0.0, 0.0, 1e-40], np.float32)
    a = np.array([0.0, 1e-30, -1e-35, 1e20, 1e-10, 5.0, 1.0, -1.0, 1e-30], np.float32)
    ra = rng.uniform(-10, 10, 4096).astype(np.float32)
    rb = rng.uniform(0.1, 10, 4096).astype(np.float32) * rng.choice([-1, 1], 4096).astype(np.float32)
    return np.concatenate([a, ra]), np.concatenate([b, rb])


def _nz(w):
    """safe_mul(w, 1): the gradient a unit seed leaves (an exact zero weight gives +0)."""
    return np.where(w == 0, np.float32(0), w).astype(np.float32)


def _ulp(a, b):
    ai = a.view(np.int32).astype(np.int64); bi = b.view(np.int32).astype(np.int64)
    ai = np.where(ai < 0, -(ai & 0x7fffffff), ai); bi = np.where(bi < 0, -(bi & 0x7fffffff), bi)
    return np.abs(ai - bi)


OPS = ["add", "sub", "mul", "div", "neg", "sin", "cos", "exp", "log", "sqrt", "rcp", "abs", "fmadd", "hsum"]


def _partials(ek, op, xs):
    """(FloatD inputs, output builder, [reference partial per input (float32, from the backend's own primal
    values)], [float64 analytic partial per input], [bound per input: ('ulp', k) or ('abs', e)])."""
    from enoki_b200 import autodiff as ad
    f32 = np.float32
    prim = lambda f, *a: f(*[ek.Float32.copy(v) for v in a]).numpy()
    d = [x.astype(np.float64) for x in xs]
    if op == "add":
        return lambda a, b: a + b, [np.ones_like(xs[0]), np.ones_like(xs[0])], [1.0, 1.0], [("ulp", 0)] * 2
    if op == "sub":
        return lambda a, b: a - b, [np.ones_like(xs[0]), -np.ones_like(xs[0])], [1.0, -1.0], [("ulp", 0)] * 2
    if op == "mul":
        return lambda a, b: a * b, [xs[1], xs[0]], [d[1], d[0]], [("ulp", 0)] * 2
    if op == "div":
        rb = prim(ek.rcp, xs[1])
        return (lambda a, b: a / b, [rb, -xs[0] * (rb * rb)], [1 / d[1], -d[0] / (d[1] * d[1])],
                [("ulp", 1), ("ulp", 4)])
    if op == "neg":
        return lambda a: -a, [np.full_like(xs[0], -1)], [-1.0], [("ulp", 0)]
    if op == "sin":
        return ad.sin, [prim(ek.cos, xs[0])], [np.cos(d[0])], [("abs", 1.2e-7)]
    if op == "cos":
        return ad.cos, [-prim(ek.sin, xs[0])], [-np.sin(d[0])], [("abs", 1.2e-7)]
    if op == "exp":
        return ad.exp, [prim(ek.exp, xs[0])], [np.exp(d[0])], [("ulp", 3)]
    if op == "log":
        return ad.log, [prim(ek.rcp, xs[0])], [1 / d[0]], [("ulp", 1)]
    if op == "sqrt":
        return ad.sqrt, [f32(0.5) / prim(ek.sqrt, xs[0])], [0.5 / np.sqrt(d[0])], [("ulp", 2)]
    if op == "rcp":
        r = prim(ek.rcp, xs[0])
        return ad.rcp, [-(r * r)], [-1 / (d[0] * d[0])], [("ulp", 3)]
    if op == "abs":
        return ad.abs_, [np.copysign(f32(1), xs[0])], [np.sign(d[0])], [("ulp", 0)]
    if op == "fmadd":
        return ad.fmadd, [xs[1], xs[0], np.ones_like(xs[0])], [d[1], d[0], 1.0], [("ulp", 0)] * 3
    if op == "hsum":
        return ad.hsum, [np.ones_like(xs[0])], [1.0], [("ulp", 0)]
    raise ValueError(op)


@pytest.mark.parametrize("backward", [True, False], ids=["backward", "forward"])
@pytest.mark.parametrize("op", OPS)
def test_floatd_partials(gpu, op, backward):
    """Each FloatD op's gradient, (1) bit for bit against a float32 restatement of the reference's partial on the
    backend's own primal values and (2) against the float64 analytic derivative within the accuracy the primal
    op is held to (test_gpu_eval.py), where that derivative is finite and normal in float32."""
    ek = gpu
    from enoki_b200 import autodiff as ad
    rng = np.random.default_rng(OPS.index(op))
    x = _inputs(rng)
    if op in ("log", "sqrt"):
        x = np.abs(x)
    if op == "div":
        xs = list(_div_pairs(rng))
    elif op in ("add", "sub", "mul"):
        xs = [x, rng.permutation(x)]
    elif op == "fmadd":
        xs = [x, rng.permutation(x), rng.permutation(x)]
    else:
        xs = [x]
    f, ref, exact, bounds = _partials(ek, op, xs)
    n = len(xs[0])
    for i in range(len(xs)):
        ins = [ad.FloatD(ek.Float32.copy(v)) for v in xs]
        for v in ins:
            ad.set_requires_gradient(v)
        y = f(*ins)
        if backward:
            ad.backward(y)
            got = np.broadcast_to(ad.gradient(ins[i]).numpy(), (n,))
            want = np.broadcast_to(_nz(np.asarray(ref[i], np.float32)), (n,))
        else:
            ad.forward(ins[i])
            got = ad.gradient(y).numpy()
            want = _nz(np.asarray(ref[i], np.float32))
            if op == "hsum":                          # a size-1 target sums the wide product
                want = np.array([np.float32(n)])
        assert_same(np.ascontiguousarray(got), np.ascontiguousarray(want), f"{op} d/dx{i}")
        if op == "hsum" and not backward:
            continue
        e = np.broadcast_to(np.asarray(exact[i], np.float64), (n,))
        with np.errstate(all="ignore"):
            ok = np.isfinite(e) & (np.abs(e) >= np.finfo(np.float32).tiny) & (np.abs(e) <= np.finfo(np.float32).max)
            if op in ("sin", "cos"):
                ok &= np.abs(xs[0]) <= 8192
            if op == "abs":
                ok &= xs[0] != 0
            if op == "div":
                r2 = 1 / (xs[1].astype(np.float64) ** 2)
                ok &= (r2 >= np.finfo(np.float32).tiny) & (r2 <= np.finfo(np.float32).max)
        kind, tol = bounds[i]
        g32, e32 = np.ascontiguousarray(got[ok]), e[ok].astype(np.float32)
        if kind == "ulp":
            assert _ulp(g32, e32).max(initial=0) <= tol, (op, i, xs[0][ok][np.argmax(_ulp(g32, e32))])
        else:
            assert np.abs(g32.astype(np.float64) - e[ok]).max(initial=0) <= tol, (op, i)
