"""CPU tests of the zstd search class compressing against a dictionary (zmt_zstd_compress_dict_device's rule,
zstd_lazy_rule.h): the C twin (zlazy_dict_twin.c) equals the Python restatement (_zdictenc.sequences) sequence for
sequence on trained, finalized and raw-content dictionaries; a corpus reaches, and asserts that it reaches, each edge of
the walk; the twin's framed streams are restored by libzstd's ZSTD_decompress_usingDict, with Dictionary_ID fields of 1,
2 and 4 bytes; and a trained dictionary makes the records' frames smaller.  No GPU."""
import numpy as np
import pytest

import _zdict as zd
import _zdictenc as zde
import _zlazy as zl

EDGE = {name: i for i, name in enumerate(zde.EDGES)}


def rows(blocks):
    return [np.asarray(b, np.int64).reshape(-1, 3) for b in blocks]


def same_both_ways(src, level, D, W=None, stats=None):
    """The twin and the restatement agree (sequences and edge counts); returns the twin's blocks."""
    st_c, st_py = np.zeros(len(zde.EDGES), np.uint64), np.zeros(len(zde.EDGES), np.int64)
    a = zde.twin_sequences(src, level, D, W=W or 0, stats=st_c)
    b = zde.sequences(src, level, D, W=W, stats=st_py)
    assert len(a) == len(b)
    for k, (x, y) in enumerate(zip(rows(a), rows(b))):
        assert np.array_equal(x, y), "block %d differs at level %d" % (k, level)
    assert st_c.astype(np.int64).tolist() == st_py.tolist()
    assert zde.replay(src, b, D) == np.ascontiguousarray(src, np.uint8).tobytes()
    if stats is not None:
        stats += st_py
    return a


def record_chunk(seed, n):
    return np.concatenate(zd.records(seed, 40))[:n]


@pytest.mark.parametrize("level", [6, 9, 12])
@pytest.mark.parametrize("kind", ["trained", "finalized", "raw"])
def test_twin_equals_restatement_on_dictionaries(kind, level):
    if kind == "trained":
        d = zd.train(7, 16 << 10)
    elif kind == "finalized":
        d = zd.finalize(9, np.concatenate(zd.records(10, 60))[: 12 << 10], 16 << 10, level=9, dict_id=300)
    else:
        d = np.concatenate(zd.records(11, 40))[: 12 << 10]
    D = zde.content(d)
    assert (D.size < d.size) == (kind != "raw")
    st = np.zeros(len(zde.EDGES), np.int64)
    same_both_ways(record_chunk(5, 20000), level, D, stats=st)
    assert st[EDGE["switch_after_0"]] > 0


def test_no_dictionary_is_the_rule_without_one():
    src = record_chunk(6, 20000)
    for level in (6, 12):
        want = zl.twin_sequences(src, level)
        for D in (None, np.zeros(0, np.uint8), np.frombuffer(b"abc", np.uint8)):      # empty, shorter than minMatch
            assert all(np.array_equal(x, y) for x, y in zip(zde.twin_sequences(src, level, D), want))
            same_both_ways(src, level, D)
        assert all(np.array_equal(x, y) for x, y in zip(rows(zl.sequences(src, level)), rows(zde.sequences(src, level))))


def test_empty_chunk():
    D = np.frombuffer(b"hello dictionary", np.uint8)
    assert zde.twin_sequences(np.zeros(0, np.uint8), 6, D) == [] and zde.sequences(np.zeros(0, np.uint8), 6, D) == []


def rand(rng, n):
    return rng.integers(0, 256, n).astype(np.uint8)


def test_edges_of_the_walk():
    """Each edge of the walk, reached by a constructed chunk and checked on both restatements."""
    rng = np.random.default_rng(1)
    st = np.zeros(len(zde.EDGES), np.int64)
    # chain switches after depth - 1 chunk steps, and never (depth used up in the chunk): level 6 walks 8 steps
    key = np.frombuffer(b"KEYWORD-", np.uint8)
    parts = []
    for _ in range(10):
        parts += [key, rand(rng, 24)]
    D = np.concatenate([rand(rng, 300), key, rand(rng, 300)])
    same_both_ways(np.concatenate(parts), 6, D, stats=st)
    assert st[EDGE["switch_after_depth_minus_1"]] > 0 and st[EDGE["depth_used_in_chunk"]] > 0

    # distances W (taken) and W + 1 (not taken): raw content larger than level 6's 2 MiB window
    W = zl.window(6)
    D = rand(rng, W + 4096)
    dlen = D.size
    src = rand(rng, 1024)
    src[0:64] = D[dlen - W: dlen - W + 64]                               # p = 0: distance 0 + dlen - q = W
    src[300:364] = D[dlen + 300 - (W + 1): dlen + 300 - (W + 1) + 64]    # p = 300: distance W + 1
    s0 = st.copy()
    blocks = same_both_ways(src, 6, D, stats=st)
    offs = np.concatenate([b[:, 1] for b in rows(blocks)])
    assert (offs == W).any() and (offs <= W).all()
    assert st[EDGE["dist_W"]] > s0[EDGE["dist_W"]] and st[EDGE["dist_W_plus_1"]] > s0[EDGE["dist_W_plus_1"]]

    # a match cut at the dictionary's end, then a longer candidate further back; and the skip bl >= dlen - q
    P = rand(rng, 96)
    D = np.concatenate([rand(rng, 200), P, rand(rng, 200), P[:20]])      # nearest: P's head at the very end of D
    s0 = st.copy()
    blocks = same_both_ways(np.concatenate([rand(rng, 50), P, rand(rng, 50)]), 9, D, stats=st)
    assert st[EDGE["capped_then_longer"]] > s0[EDGE["capped_then_longer"]]
    assert any(int(ml) >= 96 for _, _, ml in rows(blocks)[0])           # the whole of P, from the farther copy
    Q = rand(rng, 40)
    D = np.concatenate([rand(rng, 100), Q[:10]])
    s0 = st.copy()
    same_both_ways(np.concatenate([Q, rand(rng, 30), Q, rand(rng, 30)]), 9, D, stats=st)
    assert st[EDGE["skip_at_dict_end"]] > s0[EDGE["skip_at_dict_end"]]
    assert (st > 0).all(), dict(zip(zde.EDGES, st.tolist()))


def frame_dict_id(frame):
    fhd = int(frame[4])
    dl = {0: 0, 1: 1, 2: 2, 3: 4}[fhd & 3]
    return dl, int.from_bytes(bytes(frame[5: 5 + dl]), "little")


@pytest.mark.parametrize("level", [6, 12])
def test_framed_streams_restored_by_libzstd(level):
    recs = zd.records(31, 12)
    chunk = 4096
    src = np.zeros(len(recs) * chunk, np.uint8)
    cb = np.array([r.size for r in recs], np.uint32)
    for i, r in enumerate(recs):
        src[i * chunk: i * chunk + r.size] = r
    content = np.concatenate(zd.records(32, 60))[: 20 << 10]
    dicts = [("trained", zd.train(7, 16 << 10)), ("raw", content)]
    dicts += [("id_%d" % i, zd.finalize(9, content, 24 << 10, level=9, dict_id=i)) for i in (7, 300, 70000)]
    for name, d in dicts:
        did = zd.dict_id(d)
        stream = zde.framed_b200(src, chunk, level, cb, zde.content(d), did)
        frames = zde.frames(stream)
        assert len(frames) == len(recs)
        for f, r in zip(frames, recs):
            assert frame_dict_id(f) == (zde.did_bytes(did), did), name
            bad, out = zd.decompress(f, d, r.size)
            assert not bad and np.array_equal(out, r), name
    assert [zde.did_bytes(i) for i in (0, 7, 300, 70000)] == [0, 1, 2, 4]


def test_trained_dictionary_makes_records_smaller():
    recs = zd.records(41, 64, lo=1024, hi=4096)
    chunk = 4096
    src = np.zeros(len(recs) * chunk, np.uint8)
    cb = np.array([r.size for r in recs], np.uint32)
    for i, r in enumerate(recs):
        src[i * chunk: i * chunk + r.size] = r
    d = zd.train(7, 32 << 10)
    with_d = zde.framed_b200(src, chunk, 9, cb, zde.content(d), zd.dict_id(d)).size
    without = zde.framed_b200(src, chunk, 9, cb).size
    assert with_d < without, (with_d, without)
