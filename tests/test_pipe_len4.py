"""The chain walks of the LZ4 level-1 compressor (and of the zstd level-3 encoder on the same front end) measure a
candidate piece in one compare (c_piece_len4): the 4 known bytes skipped, one 16-byte window at the start and one at
the offset, a mismatch scan capped at min(cut, limit).  The schedule rests on that length being a function of the
piece's start q alone (its offset, the cut at the first segment boundary that leaves it >= 4 bytes, limit = n - 5):
walk 1's chains write the same PipeTile::len4 nibble where they meet, and the back end reads the nibble instead of
measuring again.  This test restates the measure from q alone in numpy and checks, on the edge corpus of
tests/_pipecorpus.py and on generated blocks, that it fits in the window (at most 15 bytes past the known 4) and equals,
nibble for nibble, the length the schedule model's walks measure at every position a walk takes.  No GPU involved."""
from collections import defaultdict

import numpy as np
import pytest

import _pipecorpus as pc
import _pipesched as ps
import zstdmt_b200 as z


def piece_len4(s, n, off):
    """L - 4 of the candidate piece at every position of the block from its start alone (0 where there is no
    candidate): the 4 known bytes skipped, then the bytes that still match at offset off[q], up to min(cut, limit)."""
    q = np.flatnonzero(off)
    out = np.zeros(n, np.int64)
    if q.size == 0:
        return out
    d = off[q]
    B = (q & ~(ps.C_SEG - 1)) + ps.C_SEG
    B = np.where(B - q < 4, B + ps.C_SEG, B)
    cap = np.minimum(B, n - 5) - (q + 4)
    assert (cap >= 0).all() and (cap <= 15).all()
    b = np.frombuffer(bytes(s), np.uint8)
    agree = np.ones(q.size, bool)
    L = np.zeros(q.size, np.int64)
    for j in range(15):
        agree &= (j < cap) & (b[q + 4 + j] == b[q + 4 + j - d])
        L += agree
    out[q] = L
    return out


def walk_lengths(src, monkeypatch):
    """Runs the model on one block; returns (the block's offsets, {block position: L - 4 as a walk measured it})."""
    seen = defaultdict(set)
    nib = ps.Tile.nib

    def record(self, qr, L, mode):
        seen[self.t0 + qr].add(L - 4)
        return nib(self, qr, L, mode)

    monkeypatch.setattr(ps.Tile, "nib", record)
    _, _, off, _ = ps.lz4_block(src)
    monkeypatch.undo()
    return off, seen


def check_block(src, monkeypatch):
    n = len(src)
    s = bytes(np.asarray(src, np.uint8).tobytes()) + bytes(40)
    off, seen = walk_lengths(src, monkeypatch)
    ln = piece_len4(s, n, off)
    for p, vals in seen.items():
        assert off[p] != 0, ("a walk took a position without a candidate", p)
        assert vals == {int(ln[p])}, ("the length from the start alone differs from the walks' length", p, sorted(vals), int(ln[p]))
    return len(seen)


@pytest.mark.parametrize("name", [b.__name__ for b in pc.BUILDERS])
def test_piece_len4_matches_walks_on_corpus(name, monkeypatch):
    src, chunk, marks, _ = dict((b.__name__, b) for b in pc.BUILDERS)[name]()
    taken = 0
    for part in pc.parts(src, chunk, marks):
        for b0 in range(0, len(part), ps.BLK):
            taken += check_block(part[b0: b0 + ps.BLK], monkeypatch)
    if name not in ("tiny_blocks",):
        assert taken > 0, "no walk took a candidate piece"


@pytest.mark.parametrize("kind", ["mix", "text", "zeros", "random"])
def test_piece_len4_matches_walks_on_generated(kind, monkeypatch):
    chunk = 1 << 20
    gen = {"mix": z.GEN_MIX, "text": z.GEN_TEXT, "zeros": z.GEN_ZEROS, "random": z.GEN_RANDOM}[kind]
    data = z.gen_stream(gen, 2 * chunk, chunk)
    taken = 0
    for b0 in (0, chunk - ps.BLK, chunk + 5 * ps.BLK):             # first and last block of a chunk, one inside
        taken += check_block(data[b0: b0 + ps.BLK], monkeypatch)
    if kind != "random":
        assert taken > 0, "no walk took a candidate piece"
