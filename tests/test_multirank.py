"""CPU test of the N>1 path (no collective on the data path): world_size-2 gloo processes each own the chunks
`rank, rank+2, ...` (what bench.py --gpus N and ZSTDMT_GPUS do), frame them independently, and the frames
re-serialised by global chunk index must equal the single-process stream byte for byte (SURVEY.md fact 0.7:
output is independent of how chunks are dealt).  The per-rank "codec" here is the oracle's CPU twin of the GPU
encoder (tests only); what is under test is the dealing + reassembly logic and the generator's (first, stride)."""
import os
import sys

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHUNK, NCHUNKS, WORLD = 256 << 10, 9, 2


def _worker(rank, port, tmpdir):
    sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import _oracle as o
    import zstdmt_b200 as z
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=WORLD)
    mine = [i for i in range(NCHUNKS) if i % WORLD == rank]
    shard = z.gen_stream(z.GEN_MIX, len(mine) * CHUNK, CHUNK, first=rank, stride=WORLD)
    framed = o.orc_encode_lz4(shard, CHUNK)
    offs, sizes = z.scan_frames(framed)
    assert len(offs) == len(mine)
    # whole-job byte counts, the way bench.py aggregates `value` (sum over ranks)
    t = torch.tensor([shard.size, framed.size], dtype=torch.int64)
    dist.all_reduce(t)
    np.save(os.path.join(tmpdir, "framed_%d.npy" % rank), framed)
    np.save(os.path.join(tmpdir, "tot_%d.npy" % rank), t.numpy())
    dist.barrier()
    dist.destroy_process_group()


def test_round_robin_reassembly_world2(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import _oracle as o
    import zstdmt_b200 as z
    port = 29500 + (os.getpid() % 2000)
    mp.start_processes(_worker, args=(port, str(tmp_path)), nprocs=WORLD, join=True, start_method="spawn")
    whole = z.gen_stream(z.GEN_MIX, NCHUNKS * CHUNK, CHUNK)
    expect = o.orc_encode_lz4(whole, CHUNK)
    per_rank = []
    for r in range(WORLD):
        fr = np.load(os.path.join(str(tmp_path), "framed_%d.npy" % r))
        offs, sizes = z.scan_frames(fr)
        per_rank.append([fr[int(a): int(a) + 12 + int(s)] for a, s in zip(offs, sizes)])
    # in-order writer: frame i comes from rank i % WORLD (the pt_write rule, lz4-mt_compress.c:186-202)
    merged = np.concatenate([per_rank[i % WORLD][i // WORLD] for i in range(NCHUNKS)])
    assert merged.size == expect.size and np.array_equal(merged, expect)
    tot = np.load(os.path.join(str(tmp_path), "tot_0.npy"))
    assert int(tot[0]) == NCHUNKS * CHUNK and int(tot[1]) == expect.size
    rc, back = o.orc_decode(o.CODEC_LZ4, merged, whole.size)
    assert rc == 0 and np.array_equal(back, whole)


def test_dealt_streams_partition_the_global_stream_in_batches():
    """bench.py deals chunks in batches of 8 (the product's slot granularity): rank r's share is
    zmt_gen_stream_dealt(rank, world, batch); the shares must tile the one global stream, and every rank must see every
    data class of the mix (the round-1 bench aliased class = chunk index mod 8 with rank = chunk index mod N)."""
    import zstdmt_b200 as z
    chunk, batch = 1 << 16, 8
    for world in (1, 2, 4, 8):
        per = 4 * batch                                             # chunks per rank
        glob = z.gen_stream(z.GEN_MIX, per * world * chunk, chunk)
        for r in range(world):
            mine = z.gen_stream(z.GEN_MIX, per * chunk, chunk, deal=(r, world, batch))
            for i in range(per):
                g = (i // batch) * batch * world + r * batch + i % batch
                assert np.array_equal(mine[i * chunk:(i + 1) * chunk], glob[g * chunk:(g + 1) * chunk]), (world, r, i)
            classes = {((i // batch) * batch * world + r * batch + i % batch) & 7 for i in range(per)}
            assert classes == set(range(8))
