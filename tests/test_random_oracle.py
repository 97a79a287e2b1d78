"""CPU checks of the device draws of the prover's random polynomials (K26, csrc/chacha.cuh, h2_poly_random): the oracle's two
restatements of the ChaCha20Rng keystream and of Field::random (oracle/chacha.py) against known vectors and each other, the
emulated kernel body against the oracle, its 512-bit reduction on the inputs random keystream never reaches, the library's
refusals on the ABI stand-in (tests/fake_random.py), and whole proofs drawn through halo2_b200.ChaCha20Rng against the
oracle's provers under HostChaCha20Rng."""
import ctypes
import random

import numpy as np
import pytest

from oracle import chacha as C
from oracle import cref, pasta
from tests import fake_random
from tests import plonk_api_circuit as circ
from tests import plonk_prover as PP
from tests import plonk_verifier as PV
from tests import prover_replay as R
from tests.kernel_emul import build as emul_build

FIELDS = ("fp", "fq")
# RFC 8439 appendix A.1, test vector #1 (zero key, zero nonce, counter 0): the keystream's first 16 bytes
RFC8439_A1_1 = bytes.fromhex("76b8e0ada0f13d90405d6ae55386bd28")
# rand_chacha 0.3.1's test_chacha_true_values_a: ChaCha20Rng::from_seed([0; 32]), 32 next_u32
RAND_CHACHA_TRUE_VALUES_A = [
    0xade0b876, 0x903df1a0, 0xe56a5d40, 0x28bd8653, 0xb819d2bd, 0x1aed8da0, 0xccef36a8, 0xc70d778b,
    0x7c5941da, 0x8d485751, 0x3fe02477, 0x374ad8b8, 0xf4b8436a, 0x1ca11815, 0x69b687c3, 0x8665eeb2,
    0xbee7079f, 0x7a385155, 0x7c97ba98, 0x0d082d73, 0xa0290fcb, 0x6965e348, 0x3e53c612, 0xed7aee32,
    0x7621b729, 0x434ee69c, 0xb03371d5, 0xd539d874, 0x281fed31, 0x45fb0a51, 0x1f0ae1ac, 0x6f4d794b,
]
# OpenSSL's ChaCha20 (through the `cryptography` package) on random keys: one 64-byte block with the 16-byte IV
# counter (8 bytes LE) || stream (8 bytes LE) -- rand_chacha's state words 12-15.  (counter, stream, key, block)
OPENSSL_BLOCKS = [
    (0, 0, "52f22665a60c12d289185d950ee8813609166f6b113d178d6c0fd3901ff239a1",
     "6af4e41e9fb7cc5c9c92bf78f8d56898c6aa669dca3372a81a454ee8887ddb859da15c8dbe6ad7b2db04c4a4ae78eea617f845af4a841be6b7058cfa79f1d1de"),
    (5, 0, "a095f20f9395650cf9380b8edb224a6b248a1e924e8fd0ae2e1a9492a3305f18",
     "a696610582501e863b0e7b8aabd042b6b0330d4579f2f6282660f250b84a4b4f8e6d0f61a1e3bb0f263b67bb0152fab234ddded8112d85302e9c6b203477ddff"),
    ((1 << 32) - 1, 0, "8cb610900f9e347fae886dc6507795ec745c4c3fcb2eb2c73e14934c867ee057",
     "d3435f16bba4d123ab8b2d6326f720f25c84fc2b9c37546492d0580abec8a60e3e70faccf7913042a505e1c47c91961100ffa2650cfb9e562ed37c4f981bd6d0"),
    (1 << 32, 0, "ba72499bfa121e836b2ac15726ee7d6b0af6ab13c38e92cae0d15057b159987f",
     "e4bdc4873e0b1f8d376a047cf8d0ba01150ada2624ab0f6c51a7731e03dc761f52829ecc0170a1a3abb15e9a8724faf26a9e038e508130ace968ef9400616bdb"),
    ((1 << 32) - 1, (1 << 40) + 7, "94cc7411d717f14579b2aa100fbbb34fa593feaed27248b762e3ab5805f0765a",
     "4c1b45fb1c58f9e099e217e4255454469f7cfc918db09f8ef22eb2b0cb01a27ae18467bc7fe995039f95ac86637ae846d765a43abe42817174e8aaa1ef7a2c4e"),
    (0, 0x0123456789ABCDEF, "2b9c1d7e0f37c44921bd3f6564eadf7f142a72668c47e223d16edd8c47b46afc",
     "bc07cda20003f8652a7b62b7ba35759ba131706058975787963667114cc3d43c43dd3b484fcf7e3438637d482cf57fcc42d4eca8ba930cd153ed85964c1c4bc9"),
]


def _words_bytes(words) -> bytes:
    return b"".join(int(w).to_bytes(4, "little") for w in words)


def _seed(rnd) -> bytes:
    return bytes(rnd.getrandbits(8) for _ in range(32))


def _ints(b) -> list:
    return [int.from_bytes(r.tobytes(), "little") for r in b]


@pytest.fixture(scope="module")
def emu():
    lib = ctypes.CDLL(emul_build.build())
    for name in ("emu_chacha_block", "emu_chacha_reduce", "emu_chacha_random"):
        getattr(lib, name).restype = None
    return lib


def _emu_random(emu, field, seed, stream, word_pos, lens):
    out = np.zeros((sum(lens), 32), dtype=np.uint8)
    emu.emu_chacha_random(cref.FIELD_ID[field], ctypes.c_char_p(seed), ctypes.c_uint64(stream), ctypes.c_uint64(word_pos // 16),
                          ctypes.c_uint32(word_pos % 16), ctypes.c_uint64(len(lens)), (ctypes.c_uint64 * len(lens))(*lens), cref._p(out))
    return out


def test_keystream_known_vectors(emu):
    zero = bytes(32)
    for words in (C.py_words(zero, 0, 0, 32), list(C.keystream_words(zero, 0, 0, 32))):
        assert _words_bytes(words[:4]) == RFC8439_A1_1
        assert words == RAND_CHACHA_TRUE_VALUES_A
    out = np.zeros(16, dtype=np.uint32)
    emu.emu_chacha_block(ctypes.c_char_p(zero), ctypes.c_uint64(0), ctypes.c_uint64(1), out.ctypes.data_as(ctypes.c_void_p))
    assert list(out) == RAND_CHACHA_TRUE_VALUES_A[16:]
    # every word position reads the same stream
    assert C.py_words(zero, 0, 13, 19) == RAND_CHACHA_TRUE_VALUES_A[13:]


@pytest.mark.parametrize("counter,stream,key,block", OPENSSL_BLOCKS)
def test_keystream_matches_openssl_blocks(emu, counter, stream, key, block):
    key = bytes.fromhex(key)
    assert _words_bytes(C.py_block(key, stream, counter)).hex() == block
    assert _words_bytes(C.keystream_words(key, stream, 16 * counter, 16)).hex() == block
    out = np.zeros(16, dtype=np.uint32)
    emu.emu_chacha_block(ctypes.c_char_p(key), ctypes.c_uint64(stream), ctypes.c_uint64(counter), out.ctypes.data_as(ctypes.c_void_p))
    assert _words_bytes(out).hex() == block


def test_keystream_matches_the_cryptography_package():
    """The same on fresh random keys, where the `cryptography` package is importable."""
    pytest.importorskip("cryptography")
    from cryptography.hazmat.primitives.ciphers import Cipher, algorithms
    rnd = random.Random(11)
    for counter in (0, 5, (1 << 32) - 1, 1 << 32, (1 << 63) + 3):
        for stream in (0, (1 << 40) + 7, (1 << 64) - 1):
            key = _seed(rnd)
            iv = counter.to_bytes(8, "little") + stream.to_bytes(8, "little")
            want = Cipher(algorithms.ChaCha20(key, iv), mode=None).encryptor().update(bytes(64))
            assert _words_bytes(C.keystream_words(key, stream, 16 * counter, 16)) == want, (counter, stream)


@pytest.mark.parametrize("field", FIELDS)
def test_c_oracle_equals_python_oracle(field):
    rnd = random.Random(5 if field == "fp" else 6)
    for word in range(16):
        for block in (0, 7, (1 << 32) - 2):
            seed, stream = _seed(rnd), rnd.choice([0, (1 << 40) + 7])
            p = 16 * block + word
            assert _ints(C.draws(field, seed, stream, p, 5)) == C.py_draws(field, seed, stream, p, 5), (word, block)
    seed = _seed(rnd)
    p = 16 * ((1 << 32) - 2048) + 9                                # 2^12 draws across counter 2^32
    assert _ints(C.draws(field, seed, 3, p, 1 << 12)) == C.py_draws(field, seed, 3, p, 1 << 12)


@pytest.mark.parametrize("field", FIELDS)
def test_emulated_kernel_equals_oracle(emu, field):
    rnd = random.Random(21 if field == "fp" else 22)
    for word in range(16):
        for block in (0, (1 << 32) - 3):
            seed, stream = _seed(rnd), rnd.choice([0, (1 << 40) + 7])
            lens = [1, 17, 0, 9]
            want = C.draws(field, seed, stream, 16 * block + word, sum(lens))
            assert (_emu_random(emu, field, seed, stream, 16 * block + word, lens) == want).all(), (word, block)
    seed = _seed(rnd)
    assert (_emu_random(emu, field, seed, 0, 16 * 5 + 3, [1 << 12]) == C.draws(field, seed, 0, 16 * 5 + 3, 1 << 12)).all()


def _structured_u512(m: int):
    top = (1 << 512) - 1
    vals = [0, 1, top, m - 1, m, m + 1, (1 << 256) - 1, 1 << 256, top - m]
    for t in (1, 2, 3, 4, 5, (1 << 256) // m, (1 << 256) // m + 1, 1 << 200, (1 << 256) - 1, top // m - 1, top // m):
        vals += [t * m - 1, t * m, t * m + 1]
    for lo in (0, m - 1, m, m + 1, 2 * m, 3 * m, 3 * m + 5, (1 << 256) - 1):   # halves >= m, and at the top of their range
        for hi in (0, 1, m - 1, m, 2 * m + 1, 3 * m, (1 << 256) - 1):
            vals.append(lo + (hi << 256))
    return [v for v in vals if 0 <= v <= top]


@pytest.mark.parametrize("field", FIELDS)
def test_reduction_on_structured_inputs(emu, field):
    m = pasta.FIELDS[field]
    vals = _structured_u512(m)
    data = np.frombuffer(b"".join(v.to_bytes(64, "little") for v in vals), dtype=np.uint8).reshape(-1, 64).copy()
    out = np.zeros((len(vals), 32), dtype=np.uint8)
    emu.emu_chacha_reduce(cref.FIELD_ID[field], cref._p(data), ctypes.c_uint64(len(vals)), cref._p(out))
    want = [v % m for v in vals]
    assert _ints(out) == want
    assert _ints(C.u512_mod(field, data)) == want
    assert [C.py_from_u512(field, [(v >> (32 * i)) & C.MASK32 for i in range(16)]) for v in vals] == want


def _handles(polys):
    return (ctypes.c_uint64 * len(polys))(*[p._h.value for p in polys])


def test_refused_calls_write_nothing():
    """Every refusal of h2_poly_random, on the stand-in that restates the library's checks: the message, and nothing written."""
    import halo2_b200
    from halo2_b200 import lib as L
    seed = bytes(range(32))
    with fake_random.installed() as fake:
        a, b, q = halo2_b200.ResidentPoly("fp", 8), halo2_b200.ResidentPoly("fp", 8), halo2_b200.ResidentPoly("fq", 8)
        sh = halo2_b200.ResidentPoly("fp", 8).share()
        for p in (a, b, q):
            p.upload(cref.ints_to_bytes(list(range(1, 9))))
        before = {h: v[1].copy() for h, v in fake.polys.items()}
        sz = lambda *xs: (ctypes.c_size_t * len(xs))(*xs)          # noqa: E731
        key = L.ptr(np.frombuffer(seed, dtype=np.uint8).copy())
        call = lambda ps, lens, k=key, block=0, word=0, count=None: fake.h2_poly_random(  # noqa: E731
            _handles(ps), ctypes.c_size_t(len(ps) if count is None else count), lens, k, ctypes.c_uint64(0), ctypes.c_uint64(block), ctypes.c_uint32(word))
        bogus = type("P", (), {"_h": ctypes.c_uint64(999999)})()
        cases = [
            (lambda: call([a], sz(8), count=0), "count == 0"),
            (lambda: fake.h2_poly_random(None, ctypes.c_size_t(1), sz(8), key, 0, 0, 0), "null argument"),
            (lambda: call([a], sz(8), k=None), "null seed32"),
            (lambda: call([a], sz(8), word=16), "word >= 16"),
            (lambda: call([bogus], sz(8)), r"polys\[0\]: unknown polynomial handle"),
            (lambda: call([a, sh], sz(8, 8)), r"polys\[1\]: the polynomial is shared"),
            (lambda: call([a, q], sz(8, 8)), r"polys\[1\]: the polynomials live in different fields"),
            (lambda: call([a, b], sz(8, 9)), r"polys\[1\]: a polynomial holds fewer than lens\[1\] elements"),
            (lambda: call([a, b, a], sz(1, 1, 1)), r"polys\[2\] is also polys\[0\]"),
            (lambda: call([a, b], sz(8, 8), block=(1 << 64) - 15), "run past keystream block"),
            (lambda: call([a], sz(1), block=(1 << 64) - 1, word=1), "run past keystream block"),
        ]
        import re
        for fn, msg in cases:
            assert fn() == 1, msg
            assert re.search(msg, fake.err.decode()), (msg, fake.err)
            assert all((fake.polys[h][1] == v).all() for h, v in before.items()), msg
        assert "h2_poly_random" not in fake.calls
        # the last block of the keystream is still reachable
        assert call([a], sz(1), block=(1 << 64) - 1) == 0 and call([a], sz(2), block=(1 << 64) - 3, word=15) == 0
        for p in (a, b, q, sh):
            p.close()


def test_device_rng_interface_on_the_stand_in():
    """halo2_b200.ChaCha20Rng: scalar() and poly(n) interleaved give HostChaCha20Rng's draws, one launch per poly(n) and one per
    batch of scalars, word_pos moving 16 per scalar; close() frees what it handed out, freed by its new owner or not."""
    import halo2_b200
    seed = bytes(range(100, 132))
    with fake_random.installed() as fake:
        for field, stream, pos in (("fp", 0, 0), ("fq", (1 << 40) + 7, 16 * ((1 << 32) - 3) + 15)):
            host = C.HostChaCha20Rng(seed, field, True, stream=stream, word_pos=pos)
            dev = halo2_b200.ChaCha20Rng(seed, field, stream=stream, word_pos=pos)
            got, want, handed = [], [], []
            for op in ("s", "p5", "s", "s", "p1", "p40", "s") + ("s",) * 300 + ("p3", "s"):
                if op == "s":
                    got.append(dev.scalar())
                    want.append(host.scalar())
                else:
                    p = dev.poly(int(op[1:]))
                    handed.append(p)
                    got += _ints(p.download())
                    want += _ints(host.poly(int(op[1:])))
                assert dev.word_pos == host.word_pos
            assert got == want
            assert fake.calls.count("h2_poly_random") == 4 + 2             # four polynomials, two batches of 256 scalars
            handed[0].close()                                       # its new owner freed it: close() leaves it alone
            dev.close()
            assert not fake.polys and all(not p._h.value for p in handed)
            fake.calls.clear()


@pytest.fixture(scope="module")
def plonk_api_setup():
    c = pasta.VESTA
    P = pasta.Params.new(c, 5)
    vk = PV.PinnedKey(circ.CASE["key_text"])
    fixed = circ.fixed_columns(circ.M, circ.ZETA)
    sigma = circ.permutation_columns(circ.M, vk.omega, circ.DELTA)
    gens = (cref.affines_to_bytes(P.g), cref.affines_to_bytes(P.g_lagrange), cref.affines_to_bytes([P.w]), cref.affines_to_bytes([P.u]))
    return c, P, vk, fixed, sigma, gens


def test_plonk_api_proof_with_the_device_rng(plonk_api_setup):
    """create_proof_engine with halo2_b200.ChaCha20Rng (random polynomial and s_poly drawn by h2_poly_random, every other
    draw through scalar()) writes the big-integer oracle prover's 4 160 bytes under HostChaCha20Rng with the same seed; the
    pinned verifier accepts them, and nothing stays allocated."""
    import halo2_b200
    c, P, vk, fixed, sigma, gens = plonk_api_setup
    seed, inst = bytes(range(7, 39)), [[[2]], [[2]]]
    W = R._WriteT(circ.M)
    PP.create_proof(c, P.g, P.g_lagrange, P.w, P.u, vk, fixed, sigma, [circ.witness(), circ.witness()], inst, C.HostChaCha20Rng(seed, "fp", False),
                    W, circ.ZETA, circ.DELTA)
    want = bytes(W.T.proof)
    assert len(want) == 4160 and PV.verify_proof(PV.OracleArm("vesta", 5, *gens), vk, want, inst, circ.DELTA)
    with fake_random.installed() as fake:
        prm = halo2_b200.Params("vesta", 5, gens[0], gens[1], gens[2], u=gens[3])
        T = R.Blake2bTranscript(circ.M)
        with halo2_b200.ChaCha20Rng(seed, "fp") as rng:
            PP.create_proof_engine(halo2_b200, prm, vk, fixed, sigma, [circ.witness(), circ.witness()], inst, rng, T, circ.ZETA, circ.DELTA)
        assert bytes(T.proof) == want
        assert fake.calls.count("h2_poly_random") >= 2 and not fake.polys
        prm.close()


@pytest.mark.parametrize("k", [4, 5, 6])
def test_benchmark_circuit_proof_with_the_device_rng(k):
    """The benchmark circuit: the engine's phase composition with halo2_b200.ChaCha20Rng writes CrefProver's bytes under
    HostChaCha20Rng; both verifiers accept, and a flipped bit is rejected."""
    import halo2_b200
    from tests import bench_circuit as BC
    c, n = pasta.VESTA, 1 << k
    pts = cref.gen_points("vesta", 99, n + 2)
    A = cref.bytes_to_affine
    P = pasta.Params.from_generators(c, k, [A(x) for x in pts[:n]], A(pts[n]), A(pts[n + 1]))
    D = pasta.EvaluationDomain("fp", BC.DEGREE, k, circ.ZETA)
    fixed, sigma, adv = BC.columns(k, circ.M, D.omega, circ.DELTA, circ.A_SMALL * circ.ZETA % circ.M)
    cl = lambda v: pasta.to_affine(c, pasta.best_multiexp(c, list(v) + [1], P.g_lagrange + [P.w]))   # noqa: E731
    vk = PV.PinnedKey(BC.pinned_key_text(k, D.extended_k, c.p, circ.M, D.omega, [cl(f) for f in fixed], [cl(s_) for s_ in sigma]))
    gens = (cref.affines_to_bytes(P.g), cref.affines_to_bytes(P.g_lagrange), cref.affines_to_bytes([P.w]), cref.affines_to_bytes([P.u]))
    adv_bytes = [cref.ints_to_bytes(col) for col in adv]
    seed = bytes([k]) * 32
    cp = PP.CrefProver(cref, "vesta", "fp", *gens, threads=4)
    Tc = R.Blake2bTranscript(circ.M)
    cp.create_proof(vk, fixed, sigma, [adv_bytes], [[]], C.HostChaCha20Rng(seed, "fp", True), Tc, circ.ZETA, circ.DELTA)
    want = bytes(Tc.proof)
    with fake_random.installed() as fake:
        prm = halo2_b200.Params("vesta", k, gens[0], gens[1], gens[2], u=gens[3])
        T = R.Blake2bTranscript(circ.M)
        with halo2_b200.ChaCha20Rng(seed, "fp") as rng:
            PP.create_proof_engine(halo2_b200, prm, vk, fixed, sigma, [adv_bytes], [[]], rng, T, circ.ZETA, circ.DELTA)
        got = bytes(T.proof)
        assert got == want
        assert not fake.polys
        earm = PV.EngineArm(halo2_b200, "vesta", k, params=prm)
        assert PV.verify_proof(earm, vk, got, [[]], circ.DELTA)
        bad = bytearray(got)
        bad[len(bad) // 3] ^= 8
        assert not PV.verify_proof(earm, vk, bytes(bad), [[]], circ.DELTA)
        earm.close()
        prm.close()
    assert PV.verify_proof(PV.OracleArm("vesta", k, *gens), vk, got, [[]], circ.DELTA)
