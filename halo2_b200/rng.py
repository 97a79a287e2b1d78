"""The prover's random polynomials drawn on the device: the scalars a seeded rand_chacha 0.3.1 ChaCha20Rng gives
pasta_curves 0.5.1's Field::random (h2_poly_random, csrc/chacha.cuh).

vanishing::Argument::commit draws its random polynomial and commitment::create_proof its s_poly, n scalars each, in a
serial loop on the host (plonk/vanishing/prover.rs:45-48, poly/commitment/prover.rs:45-48).  A draw depends only on its
keystream position, so one launch draws a whole polynomial, and a prover whose rng is a ChaCha20Rng gets the very
scalars the reference's loop would draw with it: the proof stays byte-identical.

`ChaCha20Rng` has the interface the phase calls take (`poly(n)`, `scalar()`); `random_resident` is the entry point's
wrapper."""
from __future__ import annotations

import ctypes
from typing import List, Optional, Sequence

import numpy as np

from . import lib as _l
from .poly import ResidentPoly, _handles, freed_on_failure

WORDS = 16                       # keystream words per Field::random draw (eight next_u64), and per ChaCha20 block
_POS_LIMIT = 1 << 68             # rand_chacha's block counter is 64 bits: word positions stay below 2^68


def _seed(seed) -> bytes:
    seed = bytes(seed)
    if len(seed) != 32:
        raise ValueError(f"a ChaCha20Rng seed is 32 bytes, not {len(seed)}")
    return seed


def fill_random(polys: Sequence[ResidentPoly], lens: Sequence[int], seed, stream: int = 0, word_pos: int = 0) -> None:
    """h2_poly_random: polys[i][0 .. lens[i]) <- consecutive Field::random draws of ChaCha20Rng(seed, stream) from keystream
    word position `word_pos`, polynomial i starting where polynomial i - 1 ended; one launch, asynchronous on the lane's
    stream.  Draw j reads words word_pos + 16 j ... + 15."""
    if len(polys) != len(lens):
        raise ValueError("one length per polynomial")
    if not 0 <= int(word_pos) < _POS_LIMIT:
        raise ValueError("word_pos outside [0, 2^68)")
    key = np.frombuffer(_seed(seed), dtype=np.uint8).copy()
    count = len(polys)
    _l.check(_l.init().h2_poly_random(_handles(polys), ctypes.c_size_t(count), (ctypes.c_size_t * count)(*[int(n) for n in lens]), _l.ptr(key),
                                      ctypes.c_uint64(int(stream)), ctypes.c_uint64(int(word_pos) // WORDS), ctypes.c_uint32(int(word_pos) % WORDS)))


def random_resident(field: str, lens: Sequence[int], seed, stream: int = 0, word_pos: int = 0) -> List[ResidentPoly]:
    """New resident polynomials of lens[i] elements over `field`, filled as fill_random fills them (one launch).  The
    draws cover word positions [word_pos, word_pos + 16 sum(lens))."""
    with freed_on_failure() as fresh:
        polys = [fresh.keep(ResidentPoly(field, n)) for n in lens]
        fill_random(polys, lens, seed, stream, word_pos)
    return polys


class ChaCha20Rng:
    """rand_chacha's ChaCha20Rng::from_seed(seed) with set_stream(stream) and set_word_pos(word_pos), as the prover's
    phase calls draw from it: poly(n) -> a ResidentPoly of n draws made on the device, scalar() -> int.  `word_pos`
    advances by 16 per scalar, the way a Rust ChaCha20Rng's get_word_pos() does under Field::random.

    scalar() serves from a small resident batch drawn by the same entry point and downloaded; a value depends only on its
    position, so poly(n) simply moves the position on, past the batch if need be.  The rng keeps every polynomial it hands
    out and close() frees them, whether or not their new owner freed them first (vanishing_commit's Committed does,
    opening.create_proof leaves it to the caller)."""

    BATCH = 256                  # scalars per download

    def __init__(self, seed, field: str, stream: int = 0, word_pos: int = 0):
        if field not in _l.FIELD_ID:
            raise ValueError(f"unknown field {field!r}")
        if not 0 <= int(stream) < 1 << 64:
            raise ValueError("stream outside [0, 2^64)")
        if not 0 <= int(word_pos) < _POS_LIMIT:
            raise ValueError("word_pos outside [0, 2^68)")
        self.seed, self.field, self.stream = _seed(seed), field, int(stream)
        self._pos = int(word_pos)
        self._handed: List[ResidentPoly] = []
        self._buf: Optional[ResidentPoly] = None
        self._vals: List[int] = []
        self._vals_pos = 0       # the word position of _vals[0]

    @property
    def word_pos(self) -> int:
        return self._pos

    def poly(self, n: int) -> ResidentPoly:
        """n draws into a new resident polynomial, one launch."""
        self._handed = [p for p in self._handed if p._h.value]
        p = random_resident(self.field, [int(n)], self.seed, self.stream, self._pos)[0]
        self._handed.append(p)
        self._pos += WORDS * int(n)
        return p

    def scalar(self) -> int:
        at = (self._pos - self._vals_pos) // WORDS         # the position only moves forward, 16 words at a time
        if at >= len(self._vals):
            self._refill()
            at = 0
        self._pos += WORDS
        return self._vals[at]

    def _refill(self) -> None:
        # the batch stops where the keystream does (block 2^64 - 1); past it the entry point refuses even one draw
        block, word = divmod(self._pos, WORDS)
        n = max(1, min(self.BATCH, (1 << 64) - block - (1 if word else 0)))
        if self._buf is None:
            self._buf = ResidentPoly(self.field, self.BATCH)
        fill_random([self._buf], [n], self.seed, self.stream, self._pos)
        self._vals = [int.from_bytes(r.tobytes(), "little") for r in self._buf.download(n)]
        self._vals_pos = self._pos

    def close(self) -> None:
        """Frees the scalar batch and every polynomial poly() handed out."""
        for p in self._handed:
            p.close()
        self._handed = []
        if self._buf is not None:
            self._buf.close()
            self._buf = None
        self._vals = []

    def __enter__(self) -> "ChaCha20Rng":
        return self

    def __exit__(self, *exc) -> None:
        self.close()
