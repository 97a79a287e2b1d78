"""The scalars a seeded rand_chacha 0.3.1 ChaCha20Rng gives pasta_curves 0.5.1's Field::random (TEST INFRASTRUCTURE ONLY --
see pasta.py): the oracle of the device draws (csrc/chacha.cuh, K26, h2_poly_random).

Two independent restatements: Python big integers here (py_*, for small n) and C (oracle/chacha_oracle.c, for GPU sizes),
each of the keystream -- RFC 8439's ChaCha20 block function with the seed as key, a 64-bit block counter in state words 12-13
and a 64-bit stream id in words 14-15, read word after word, little-endian -- and of from_u512: the 16 words of a draw as one
little-endian 512-bit integer, mod m.  Draw j from word position p takes words p + 16 j ... p + 16 j + 15.

HostChaCha20Rng is the host side of a prover's rng: scalar() / poly(n) in that order of draws, as tests/multiopen_cases.SeededRng
has them, so the big-integer prover and the C restatement's prover run on it unchanged."""
from __future__ import annotations

import ctypes
import os
import subprocess
from typing import List, Optional

import numpy as np

from oracle import pasta

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "chacha_oracle.c")
_SO = os.path.join(_HERE, "_build", "libchacha_oracle.so")
_lib: Optional[ctypes.CDLL] = None

FIELD_ID = {"fp": 0, "fq": 1}
WORDS = 16                      # keystream words per block, and per draw
MASK32 = 0xFFFFFFFF


def build(force: bool = False) -> str:
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
        os.makedirs(os.path.dirname(_SO), exist_ok=True)
        subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-fPIC", "-Wall", "-Wextra", "-shared", "-o", _SO, _SRC])
    return _SO


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        build()                  # no-op unless the source is newer than the library
        _lib = ctypes.CDLL(_SO)
        for name in ("orc_chacha_words", "orc_chacha_draws", "orc_u512_mod"):
            getattr(_lib, name).restype = ctypes.c_int
    return _lib


def _seed(seed: bytes) -> bytes:
    seed = bytes(seed)
    if len(seed) != 32:
        raise ValueError("a ChaCha20Rng seed is 32 bytes")
    return seed


def _split(word_pos: int):
    if not 0 <= word_pos < 1 << 68:
        raise ValueError("word position outside [0, 2^68)")
    return word_pos // WORDS, word_pos % WORDS


def _u8p(a: np.ndarray):
    return a.ctypes.data_as(ctypes.c_void_p)


# ---- C --------------------------------------------------------------------------------------------------------------
def keystream_words(seed: bytes, stream: int, word_pos: int, n: int) -> np.ndarray:
    """n keystream words from word position `word_pos`, as uint32."""
    block, word = _split(word_pos)
    out = np.zeros(n, dtype=np.uint32)
    key = np.frombuffer(_seed(seed), dtype=np.uint8).copy()
    assert lib().orc_chacha_words(_u8p(key), ctypes.c_uint64(stream), ctypes.c_uint64(block), ctypes.c_uint32(word), ctypes.c_uint64(n), _u8p(out)) == 0
    return out


def draws(field: str, seed: bytes, stream: int, word_pos: int, n: int) -> np.ndarray:
    """n Field::random draws from word position `word_pos`: (n, 32) uint8 canonical.  One thread."""
    block, word = _split(word_pos)
    out = np.zeros((n, 32), dtype=np.uint8)
    key = np.frombuffer(_seed(seed), dtype=np.uint8).copy()
    assert lib().orc_chacha_draws(FIELD_ID[field], _u8p(key), ctypes.c_uint64(stream), ctypes.c_uint64(block), ctypes.c_uint32(word),
                                  ctypes.c_uint64(n), _u8p(out)) == 0
    return out


def u512_mod(field: str, data: np.ndarray) -> np.ndarray:
    """(n, 64) uint8 little-endian 512-bit integers -> (n, 32) uint8 canonical residues mod m."""
    data = np.ascontiguousarray(data, dtype=np.uint8).reshape(-1, 64)
    out = np.zeros((data.shape[0], 32), dtype=np.uint8)
    assert lib().orc_u512_mod(FIELD_ID[field], _u8p(data), ctypes.c_uint64(data.shape[0]), _u8p(out)) == 0
    return out


# ---- Python big integers --------------------------------------------------------------------------------------------
def _rotl(x: int, n: int) -> int:
    return ((x << n) | (x >> (32 - n))) & MASK32


def py_block(seed: bytes, stream: int, block: int) -> List[int]:
    """Keystream block `block` as 16 words (RFC 8439 section 2.3; counter and stream id 64 bits each)."""
    key = _seed(seed)
    s = [int.from_bytes(b"expand 32-byte k"[4 * i:4 * i + 4], "little") for i in range(4)]
    s += [int.from_bytes(key[4 * i:4 * i + 4], "little") for i in range(8)]
    s += [block & MASK32, (block >> 32) & MASK32, stream & MASK32, (stream >> 32) & MASK32]
    x = list(s)

    def qr(a, b, c, d):
        x[a] = (x[a] + x[b]) & MASK32; x[d] = _rotl(x[d] ^ x[a], 16)      # noqa: E702
        x[c] = (x[c] + x[d]) & MASK32; x[b] = _rotl(x[b] ^ x[c], 12)      # noqa: E702
        x[a] = (x[a] + x[b]) & MASK32; x[d] = _rotl(x[d] ^ x[a], 8)       # noqa: E702
        x[c] = (x[c] + x[d]) & MASK32; x[b] = _rotl(x[b] ^ x[c], 7)       # noqa: E702
    for _ in range(10):
        qr(0, 4, 8, 12), qr(1, 5, 9, 13), qr(2, 6, 10, 14), qr(3, 7, 11, 15)
        qr(0, 5, 10, 15), qr(1, 6, 11, 12), qr(2, 7, 8, 13), qr(3, 4, 9, 14)
    return [(a + b) & MASK32 for a, b in zip(x, s)]


def py_words(seed: bytes, stream: int, word_pos: int, n: int) -> List[int]:
    block, word = _split(word_pos)
    out = []
    while len(out) < n:
        out += py_block(seed, stream, block)[word:]
        block, word = block + 1, 0
    return out[:n]


def py_from_u512(field: str, words: List[int]) -> int:
    """from_u512 of eight next_u64 made of these 16 words: the little-endian 512-bit integer mod m."""
    return sum(w << (32 * i) for i, w in enumerate(words)) % pasta.FIELDS[field]


def py_draws(field: str, seed: bytes, stream: int, word_pos: int, n: int) -> List[int]:
    w = py_words(seed, stream, word_pos, WORDS * n)
    return [py_from_u512(field, w[WORDS * j:WORDS * (j + 1)]) for j in range(n)]


class HostChaCha20Rng:
    """A prover's ChaCha20Rng on the host: scalar() -> int; poly(n) -> n draws, as ints or (n, 32) uint8 bytes (as_bytes);
    word_pos advances by 16 per scalar.  Draws through the C restatement."""

    def __init__(self, seed: bytes, field: str, as_bytes: bool, stream: int = 0, word_pos: int = 0):
        self.seed, self.field, self.as_bytes, self.stream, self.word_pos = _seed(seed), field, as_bytes, int(stream), int(word_pos)

    def _take(self, n: int) -> np.ndarray:
        b = draws(self.field, self.seed, self.stream, self.word_pos, n)
        self.word_pos += WORDS * n
        return b

    def scalar(self) -> int:
        return int.from_bytes(self._take(1)[0].tobytes(), "little")

    def poly(self, n: int):
        b = self._take(n)
        return b if self.as_bytes else [int.from_bytes(r.tobytes(), "little") for r in b]
