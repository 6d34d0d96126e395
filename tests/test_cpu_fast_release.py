"""CPU: early release in the fast sweep kernel.  The planner picks the body instruction after which the most staged input
bytes are dead; the fast lowering puts a NOP carrying FF_REL and the release mask right after what that instruction lowers
to, and the kernel refills the released inputs' buffers with the CTA's next tile there.  In the host-compiled kernel
(tests/cpu_kernel) a TMA copy is a synchronous memcpy, so a read of a released buffer after the refill, or a refill before
every thread is done with it, shows up as wrong data -- and a mis-counted mbarrier phase as a trap."""
import gc

import numpy as np

import test_cpu_emulator as base
from fast_kernel_emu import FastKernelEmulator
from test_cpu_fast_kernel import _differential

FF_REL = 0x0200                       # ek_isa.h
N = 9 * 4096 + 1000                   # 10 tiles of 4096: with 3 CTAs each strides over 3 or 4, the last tile is ragged


def _inputs(ek, n):
    from enoki_b200 import Float32
    gc.collect(); ek.lib().ek_debug_discard_side_effects(); gc.collect()
    table = {}
    F = base._Factory(Float32, table, 0x7f0000000000)
    rng = np.random.default_rng(n)
    xs = [F.copy(rng.uniform(-4, 4, n).astype(np.float32)) for _ in range(4)]
    return table, xs


def _c2(ek, x0, x1, x2, x3):
    t = ek.fmadd(x0, x1, x2)
    return ek.fmadd(ek.sin(ek.fmadd(x3, ek.exp(-(t * t)), x0)), x1, ek.sqrt(abs(t)))


def _fast_sweep(ek):
    prog = ek.debug_program()
    sw = [s for s in prog["sweeps"] if "fast" in s and s["n"] > 1]
    assert len(sw) == 1
    return prog, sw[0]


def test_c2_releases_x0_x2_x3_after_the_second_fma(ek):
    """C2's lowered body is LOAD FMA MUL EXPN FMA, then the release of x0, x2 and x3, then SIN LOAD SQRTA FMAC."""
    table, (x0, x1, x2, x3) = _inputs(ek, N)
    out = _c2(ek, x0, x1, x2, x3)
    prog, sw = _fast_sweep(ek)
    fast = sw["fast"]
    names = [prog["fops"][t[0]] for t in fast["body"]]
    rel = [k for k, t in enumerate(fast["body"]) if t[1] & FF_REL]
    fmas = [k for k, name in enumerate(names) if name.startswith("FMA")]
    assert len(rel) == 1 and rel[0] == fmas[1] + 1 and names[rel[0]] == "NOP", (names, rel)
    mask = fast["body"][rel[0]][6]
    assert mask == fast["release_mask"]
    staged = [var for var, unit, es in sw["staged"]]
    released = {staged[k] for k in range(len(staged)) if (mask >> k) & 1}
    assert released == {x0.index, x2.index, x3.index}
    del out
    ek.lib().ek_debug_discard_side_effects()


def test_early_release_on_the_host_compiled_kernel(ek, oracle, P):
    """C2 with its fused hsum and a one-input program, on the host-compiled kernel with CTAs that stride over several
    tiles and a ragged last tile, bit for bit against the numpy interpreter; C3 does not release."""
    from enoki_b200 import Float32, UInt32, gather, scatter_add, hsum
    table, (x0, x1, x2, x3) = _inputs(ek, N)
    out = _c2(ek, x0, x1, x2, x3)
    s = hsum(out)
    prog, sw = _fast_sweep(ek)
    tiles = -(-N // (sw["fast"]["T"] * 16))
    assert any(t[1] & FF_REL for t in sw["fast"]["body"]) and N % (sw["fast"]["T"] * 16) != 0
    assert tiles // min(tiles, FastKernelEmulator.max_grid) >= 3
    _differential(ek, oracle, table, {"c2": out, "sum": s}, float_tol=("sum",))
    del out, s

    # one input, released once its last reader has run; the sin / exp / multiply-add after it overlap the refill
    t = x0 * 1.5
    y = ek.fmadd(ek.sin(t), t, ek.exp(-(t * t)))
    del t
    _, sw = _fast_sweep(ek)
    assert any(t[1] & FF_REL for t in sw["fast"]["body"]) and sw["fast"]["release_mask"] == 1
    _differential(ek, oracle, table, {"y": y})
    del y

    # C3 (gather + scatter_add: bound by those, not by its stream) does not release
    U = base._Factory(UInt32, table, 0x7d0000000000)
    tab = base._Factory(Float32, table, 0x7e0000000000).copy(np.float32(0.5) + np.arange(31, dtype=np.float32) / np.float32(30))
    bins = U.copy(np.zeros(31, np.uint32))
    idx = UInt32((x0 - -4.0) * 31.0 / 8.0)
    mask = idx < UInt32(31)
    w = gather(Float32, tab, idx, mask)
    scatter_add(bins, UInt32(1), idx, mask)
    del idx, mask
    _, sw = _fast_sweep(ek)
    assert sw["fast"]["release_mask"] == 0 and not any(t[1] & FF_REL for t in sw["fast"]["body"])
    _differential(ek, oracle, table, {"bins": bins, "w": w})
    gc.collect()
