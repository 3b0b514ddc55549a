"""Host branches of the FP64 building blocks (pdq_fast.cuh, pdq_math.cuh, the per-gene tables of pdq_gene.cuh), through the
host emulator, against the high-precision references of tests/golden/math_ref.npz -- the same checks and bounds as the device
branches get in test_gpu_math.py -- and the committed lookup tables of pdq_tables.h against their definition."""
import numpy as np
import pytest

import math_checks as mc
from emu.emu_ops import EmuOps


@pytest.fixture(scope="module")
def ops():
    return EmuOps()


@pytest.mark.parametrize("name", sorted(mc.ULP_BOUNDS))
def test_host_primitive_ulp(ops, name):
    mc.check_ulp(ops, name)


@pytest.mark.parametrize("name", sorted(mc.SF_BOUNDS))
def test_host_special_function(ops, name):
    mc.check_special(ops, name)


def test_host_norm_sf(ops):
    mc.check_norm_sf(ops)


def test_host_special_inputs(ops):
    mc.check_special_inputs(ops)


def test_host_random_sweep(ops):
    worst = mc.sweep_worst(ops, 200_000)
    for name, w in worst.items():
        assert w <= mc.ULP_BOUNDS[name] + 1.0, (name, w)


@pytest.mark.parametrize("T", [1, 2, 4, 8, 16, 32])
def test_host_tables(ops, T):
    """Tables built by T emulated lanes (threads exchanging through the device's Hillis-Steele scan) within the forward-error
    bound of the recurrence, and in agreement with the single-lane build."""
    r, refs = mc.table_refs()
    out = ops.tables(r, T)
    mc.check_tables(out, r, refs, T)
    if T > 1:
        mc.check_tables_agree(out, ops.tables(r, 1), r, refs, T)


def test_committed_math_table_matches_its_definition():
    """pdq_tables.h as compiled (read back through the emulator) against scripts/gen_math_tables.py's construction, recomputed
    with mpmath: the (c, l) pairs of the log and the 2^(j/64) of the exp.  A hand-edited or stale table fails."""
    mp = pytest.importorskip("mpmath")
    mp.mp.prec = 160
    tab, lay = EmuOps().math_table()
    bits, n, split = lay["bits"], lay["n"], lay["split"]
    assert (bits, n, lay["exp_n"]) == (9, 512, 64) and tab.size == 2 * n + lay["exp_n"]
    assert split == int(mp.ceil((mp.sqrt(2) - 1) * n))

    def short(x, nbits=24):  # x rounded to nbits significant bits
        m, e = mp.frexp(x)
        return float(mp.ldexp(mp.nint(mp.ldexp(m, nbits)), e - nbits))

    def within_half_ulp(got, exact):
        return abs(mp.mpf(got) - exact) <= mp.mpf(np.spacing(abs(float(exact)))) / 2

    for i in range(n):
        c, l = tab[2 * i], tab[2 * i + 1]
        want_c = 1.0 if i == 0 else 0.5 if i == n - 1 else short(1 / (1 + (mp.mpf(i) + mp.mpf(1) / 2) / n))
        assert c == want_c, f"log table entry {i}: c = {c!r}, defined as {want_c!r}"
        # the reduction r = m c - 1 stays within 2^-10 over the interval (the first one: [0, 2^-9))
        lo_m, hi_m = 1 + mp.mpf(i) / n, 1 + mp.mpf(i + 1) / n
        assert max(abs(lo_m * c - 1), abs(hi_m * c - 1)) <= (mp.mpf(2) ** -9 if i == 0 else mp.mpf(2) ** -10)
        exact_l = -mp.log(mp.mpf(c) * (2 if i >= split else 1))
        assert within_half_ulp(l, exact_l), f"log table entry {i}: l = {l!r}, -log(c) = {exact_l}"
    for j in range(lay["exp_n"]):
        v = tab[2 * n + j]
        assert within_half_ulp(v, mp.power(2, mp.mpf(j) / 64)), f"exp table entry {j}: {v!r}"
