"""CPU tests (-m "not gpu") of the host restatement of the sequential kernel (tests/emu/emu_seq.cu, chunk_emu.seq_fibers): the bar
the GPU tests of the 1D prox's routes hold every taut-string route to.

* float64: it is the oracle's linearized / weighted taut-string, for contiguous and strided slicings.
* float32: the chunked kernel's phases (tests/emu/emu_chunked.cu, run lane by lane) scan in float arithmetic too, and must equal it bit
  for bit -- which pins the float32 chunk stitching, as test_chunk_emulation.py does for float64."""
import numpy as np

import chunk_emu
from test_chunk_emulation import cases
from vjp_emu import from_flat, to_flat


def test_emulated_cta_f32_is_bit_identical_to_sequential_f32_scan():
    """On the adversarial cases of test_chunk_emulation.py, unweighted and weighted with zero weights."""
    rng = np.random.default_rng(13)
    for y, lam in cases():
        y32 = y.astype(np.float32)
        assert np.array_equal(chunk_emu.chunked_f32(y32, lam), chunk_emu.seq_fibers(y32, 1, y32.size, 1, lam)), (y.size, lam)
        if y.size < 2:
            continue
        w = rng.uniform(0, 2 * max(lam, 0.1), y.size - 1).astype(np.float32)
        if y.size > 50:
            w[10:40] = 0.0
        assert np.array_equal(chunk_emu.chunked_f32(y32, 0.0, w), chunk_emu.seq_fibers(y32, 1, y32.size, 1, 0.0, w)), (y.size, lam, "w")


def test_sequential_f64_scan_is_the_oracle(port):
    """Fiber j of the slicing (nf, len, inc) starts at (j / inc) * inc * len + j % inc, its elements inc apart."""
    rng = np.random.default_rng(17)
    for y, lam in cases():
        assert np.array_equal(chunk_emu.seq_fibers(y, 1, y.size, 1, lam), port.tv1_linearized(y, lam)), (y.size, lam)
    for nf, ln, inc in ((6, 100, 2), (36, 70, 36), (8, 33, 4), (5, 1, 5)):
        Y = np.round(rng.normal(0, 3, (nf, ln))) + np.repeat(rng.normal(0, 2, (nf, 1)), ln, axis=1)
        W = rng.uniform(0, 2, (nf, max(ln - 1, 0)))
        W[:, ::7] = 0.0
        got = from_flat(chunk_emu.seq_fibers(to_flat(Y, inc), nf, ln, inc, 1.5), nf, ln, inc)
        gotw = from_flat(chunk_emu.seq_fibers(to_flat(Y, inc), nf, ln, inc, 0.0, to_flat(W, inc)), nf, ln, inc)
        for f in range(nf):
            assert np.array_equal(got[f], port.tv1_linearized(Y[f], 1.5)), (nf, ln, inc, f)
            assert np.array_equal(gotw[f], port.tv1_weighted(Y[f], W[f]) if ln > 1 else Y[f]), (nf, ln, inc, f, "weighted")
