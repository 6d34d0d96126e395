"""GPU: the two sweep kernels against each other.  The fast kernel for 32-bit programs (ek_sweep_fast.cu) is the default;
the general kernel (ek_sweep.cu) still runs every program that uses an operation outside the fast kernel's set, so the
battery of tests/sweep_battery.py is evaluated on both and the results must agree: bit for bit, except for float
reductions and float scatter_add totals, which the two kernels fold in different orders."""
import sys

import numpy as np
import pytest

import sweep_battery

pytestmark = pytest.mark.gpu


def test_fast_kernel_is_the_default(gpu):
    ek = gpu
    L = ek.lib()
    assert L.ek_init() == 0, L.ek_last_error()
    assert L.ek_fast_mode() == 1
    x = np.random.default_rng(5).uniform(-3, 3, 300_001).astype(np.float32)
    L.ek_stats_reset()
    y = (ek.Float32.copy(x) * 1.25 + 0.5).numpy()
    assert (y == x * np.float32(1.25) + np.float32(0.5)).all()
    st = ek.stats()
    assert int(st.sweep_launches) >= 1 and int(st.fast_launches) > 0


def _run_battery(ek, fast):
    L = ek.lib()
    L.ek_set_fast_mode(fast)
    L.ek_stats_reset()

    def evaluate(var=None):
        if var is None:
            ek.cuda_eval()
            return None
        return var.numpy()
    records = sweep_battery.battery(lambda cls, a: cls.copy(a), evaluate)
    return records, int(ek.stats().fast_launches)


def _disagreement(a, b):
    """None when the records agree, else what differs."""
    if a.array.nbytes != b.array.nbytes:
        return f"{a.name}: sizes differ"
    if a.kind == 0:
        x, y = a.array.view(np.uint8), b.array.view(np.uint8)
        diff = np.flatnonzero(x != y)
        return f"{a.name}: results differ (first at byte {diff[0]} of {x.size})" if diff.size else None
    x, y = a.array.astype(np.float64), b.array.astype(np.float64)
    finite = np.abs(x[np.isfinite(x)])
    scale = a.scale if a.scale > 0 else (finite.max() if finite.size else 0.0)
    with np.errstate(invalid="ignore"):
        ok = (np.isnan(x) & np.isnan(y)) | (x == y) | (np.abs(x - y) <= a.tol * max(scale, 1e-30))
    bad = int((~ok).sum())
    return f"{a.name}: {bad} of {x.size} values differ by more than the tolerance" if bad else None


def test_fast_and_general_kernels_agree(gpu):
    ek = gpu
    try:
        ref, general_fast_launches = _run_battery(ek, 0)
        fast, fast_launches = _run_battery(ek, 1)
    finally:
        ek.lib().ek_set_fast_mode(1)
    assert general_fast_launches == 0, "the general pass used the fast kernel"
    assert fast_launches > 0, "the fast kernel was never selected"
    assert [r.name for r in ref] == [r.name for r in fast]
    bad = [d for d in map(_disagreement, ref, fast) if d]
    sys.stderr.write(f"sweep A/B: {len(ref)} results compared, {len(bad)} disagreements, "
                     f"{fast_launches} sweeps on the fast kernel\n")
    assert not bad, "\n".join(bad)
