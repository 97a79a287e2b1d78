"""GPU tests of the device draws of the prover's random polynomials (K26, csrc/chacha.cuh, h2_poly_random) against the C
restatement of ChaCha20Rng and Field::random (oracle/chacha.py): sizes up to 2^22 in both fields, word offsets, block
counters across 2^32 and stream ids; several polynomials in one launch with their tails untouched; a lane; a shared
polynomial refused; and halo2_b200.ChaCha20Rng's interleaved scalar() / poly(n) against HostChaCha20Rng."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import chacha as C  # noqa: E402
from oracle import cref  # noqa: E402

SEED = bytes(range(0x40, 0x60))


def _draw(field, lens, seed=SEED, stream=0, word_pos=0):
    import halo2_b200
    ps = halo2_b200.random_resident(field, lens, seed, stream, word_pos)
    try:
        return [p.download() for p in ps]
    finally:
        for p in ps:
            p.close()


@pytest.mark.parametrize("field", ["fp", "fq"])
@pytest.mark.parametrize("n", [1, 17, (1 << 10) + 3, 1 << 16, 1 << 20, 1 << 22])
def test_draws_equal_the_oracle(field, n):
    word_pos = 16 * ((1 << 32) - 3) + 1 if n >= 1 << 16 else 0
    stream = (1 << 40) + 7 if n & 1 else 0
    got = _draw(field, [n], stream=stream, word_pos=word_pos)[0]
    assert (got == C.draws(field, SEED, stream, word_pos, n)).all()


@pytest.mark.parametrize("word", [0, 1, 15])
@pytest.mark.parametrize("block", [0, (1 << 32) - 3])
@pytest.mark.parametrize("stream", [0, (1 << 40) + 7])
def test_offsets_counters_and_streams(word, block, stream):
    for field in ("fp", "fq"):
        got = _draw(field, [1000], stream=stream, word_pos=16 * block + word)[0]
        assert (got == C.draws(field, SEED, stream, 16 * block + word, 1000)).all(), field


def test_several_polynomials_one_launch_tails_untouched():
    import halo2_b200
    from halo2_b200 import lib as L
    from halo2_b200.rng import fill_random
    L.init()
    lens, sizes = [300, 5, 4097], [310, 5, 5000]
    fill = [cref.gen_scalars("fq", 70 + i, s) for i, s in enumerate(sizes)]
    ps = [halo2_b200.ResidentPoly("fq", s, f) for s, f in zip(sizes, fill)]
    try:
        before = L.launch_count()
        fill_random(ps, lens, SEED, 9, 16 * ((1 << 32) - 1) + 15)
        assert L.launch_count() - before == 1
        want = C.draws("fq", SEED, 9, 16 * ((1 << 32) - 1) + 15, sum(lens))
        at = 0
        for p, n, f in zip(ps, lens, fill):
            got = p.download()
            assert (got[:n] == want[at:at + n]).all() and (got[n:] == f[n:]).all()
            at += n
    finally:
        for p in ps:
            p.close()


def test_on_a_lane_and_shared_refused():
    import halo2_b200
    from halo2_b200 import lib as L
    from halo2_b200.rng import fill_random
    L.init()
    with halo2_b200.Lane():
        assert (_draw("fp", [777], stream=3, word_pos=5)[0] == C.draws("fp", SEED, 3, 5, 777)).all()
    vals = cref.gen_scalars("fp", 5, 64)
    sh = halo2_b200.ResidentPoly("fp", 64, vals).share()
    own = halo2_b200.ResidentPoly("fp", 64, vals)
    try:
        with pytest.raises(halo2_b200.H2Error, match=r"h2_poly_random: polys\[1\]: the polynomial is shared"):
            fill_random([own, sh], [64, 64], SEED)
        with pytest.raises(halo2_b200.H2Error, match="run past keystream block"):
            fill_random([own], [2], SEED, word_pos=16 * ((1 << 64) - 1) + 1)
        with pytest.raises(halo2_b200.H2Error, match="count == 0"):
            fill_random([], [], SEED)
        assert (own.download() == vals).all() and (sh.download() == vals).all()
        lib = L.load()
        key = L.ptr(np.frombuffer(SEED, dtype=np.uint8).copy())
        hs = (ctypes.c_uint64 * 1)(own._h.value)
        assert lib.h2_poly_random(hs, ctypes.c_size_t(1), (ctypes.c_size_t * 1)(64), key, ctypes.c_uint64(0), ctypes.c_uint64(0), ctypes.c_uint32(16)) != 0
        assert lib.h2_poly_random(hs, ctypes.c_size_t(1), (ctypes.c_size_t * 1)(64), None, ctypes.c_uint64(0), ctypes.c_uint64(0), ctypes.c_uint32(0)) != 0
        assert (own.download() == vals).all()
    finally:
        own.close()
        sh.close()


def test_rng_interleaved_scalars_and_polys():
    import halo2_b200
    from halo2_b200 import lib as L
    L.init()
    for field, stream, pos in (("fp", 0, 0), ("fq", (1 << 40) + 7, 16 * ((1 << 32) - 2) + 15)):
        host = C.HostChaCha20Rng(SEED, field, True, stream=stream, word_pos=pos)
        got, want = [], []
        with halo2_b200.ChaCha20Rng(SEED, field, stream=stream, word_pos=pos) as dev:
            for op in ["s", 7, "s", "s", 1, 1 << 12, "s"] + ["s"] * 300 + [3, "s"]:
                if op == "s":
                    got.append(dev.scalar())
                    want.append(host.scalar())
                else:
                    got += [int.from_bytes(r.tobytes(), "little") for r in dev.poly(op).download()]
                    want += [int.from_bytes(r.tobytes(), "little") for r in host.poly(op)]
                assert dev.word_pos == host.word_pos
        assert got == want
