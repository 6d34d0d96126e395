"""GPU: the fast sweep kernel's early release at sizes where every CTA strides over many tiles.

With early release, the instruction after which the most staged input bytes are dead refills those inputs' buffers with
the CTA's next tile while the rest of the tile still computes, and the tile boundary issues only the rest.  The A/B
battery (test_gpu_sweep_ab.py) reaches about two tiles per CTA; here C2 (with its fused hsum) and C3 run at 2^24 + 3
elements (ragged last tile) and at 2^26 on both kernels: C2's elements and C3's integer bins must agree bit for bit,
the hsum and the float bins within the A/B test's tolerances."""
import sys

import numpy as np
import pytest

import sweep_battery
from test_gpu_sweep_ab import _disagreement

pytestmark = pytest.mark.gpu


def _run(ek, fast, x_host):
    L = ek.lib()
    L.ek_set_fast_mode(fast)
    L.ek_stats_reset()

    def evaluate(var=None):
        if var is None:
            ek.cuda_eval()
            return None
        return var.numpy()
    b = sweep_battery._Battery(lambda cls, a: cls.copy(a), evaluate)
    x = [ek.Float32.copy(a) for a in x_host]
    b.c2(x)
    for bound in (30, 31):
        b.c3(x, bound)
    del x
    return b.records, int(ek.stats().fast_launches)


@pytest.mark.parametrize("n", [(1 << 24) + 3, 1 << 26])
def test_early_release_matches_the_general_kernel(gpu, n):
    ek = gpu
    rng = np.random.default_rng(n)
    x_host = [rng.uniform(-4, 4, n).astype(np.float32) for _ in range(4)]
    try:
        ref, general_fast = _run(ek, 0, x_host)
        got, fast = _run(ek, 1, x_host)
    finally:
        ek.lib().ek_set_fast_mode(1)
    assert general_fast == 0, "the general pass used the fast kernel"
    assert fast > 0, "the fast kernel was never selected"
    assert [r.name for r in ref] == [r.name for r in got]
    bad = [d for d in map(_disagreement, ref, got) if d]
    sys.stderr.write(f"early release at n={n}: {len(ref)} results compared, {len(bad)} disagreements\n")
    assert not bad, "\n".join(bad)
