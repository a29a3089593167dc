"""The size contract of the device encoders (pytest -m gpu): an encoder writes nothing past the zmt_*c_level_workspace_bytes
bytes it is given nor past zmt_*c_out_bound bytes of output, and what the workspace held before the call does not change
its frames.  Each class runs once on an exactly sized, zeroed workspace and once on a workspace and an output that carry
a guard tail, with both filled with a non-zero pattern; the guards must come back untouched and the frames equal."""
import numpy as np
import pytest

import zstdmt_b200 as z

pytestmark = pytest.mark.gpu
GUARD = 1 << 16
CLASSES = [("lz4", 1), ("lz4", 10), ("zstd", 3), ("zstd", 6), ("zstd", 12)]
BIG = (128 << 20) + (64 << 10)           # ZL_GROUP_BYTES // BIG == 1: every chunk is a group of its own


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch


def geometry(name):
    """(src, chunk, chunk_bytes or None)"""
    if name == "one_short_chunk":
        return z.gen_stream(z.GEN_MIX, 70001, 1 << 20, first=3), 1 << 20, None
    if name == "explicit_short_chunks":
        chunk, rng = 256 << 10, np.random.default_rng(2100)
        sizes = [0, 1, 13, 65535, 65536, 65537, chunk] + [int(rng.integers(0, chunk + 1)) for _ in range(30)]
        src = z.gen_stream(z.GEN_MIX, len(sizes) * chunk, chunk, first=6)
        return src, chunk, sizes
    # two chunks of BIG bytes at most, the second one short: two groups for the chain classes
    return z.gen_stream(z.GEN_MIX, BIG + (1 << 20) + 123, 1 << 20, first=7), BIG, None


def encode(torch, codec, level, d_in, n, chunk, d_cb, nch, work, out):
    L = z.lib()
    fn = L.zmt_lz4_compress_level_device if codec == "lz4" else L.zmt_zstd_compress_level_device
    foff = torch.zeros(nch + 1, dtype=torch.int64, device="cuda")
    rc = fn(d_in.data_ptr(), n, chunk, d_cb.data_ptr() if d_cb is not None else None, nch, level,
            work.data_ptr(), out.data_ptr(), foff.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0, z.ST_NAMES.get(rc, rc)
    torch.cuda.synchronize()
    return foff


@pytest.mark.parametrize("geom", ["one_short_chunk", "explicit_short_chunks", "two_groups"])
@pytest.mark.parametrize("codec,level", CLASSES)
def test_encoder_stays_inside_its_workspace(torch, codec, level, geom):
    L = z.lib()
    src, chunk, sizes = geometry(geom)
    n = int(src.size)
    nch = len(sizes) if sizes is not None else L.zmt_chunk_count(n, chunk)
    if codec == "lz4":
        wb, ob = L.zmt_lz4c_level_workspace_bytes(nch, chunk, level), L.zmt_lz4c_out_bound(nch, chunk)
    else:
        wb, ob = L.zmt_zstdc_level_workspace_bytes(nch, chunk, level), L.zmt_zstdc_out_bound(nch, chunk)
    assert wb > 0 and ob > 0
    d_in = torch.from_numpy(src).cuda()
    d_cb = torch.from_numpy(np.asarray(sizes, np.int32)).cuda() if sizes is not None else None

    work0 = torch.zeros(wb, dtype=torch.uint8, device="cuda")
    out0 = torch.zeros(ob, dtype=torch.uint8, device="cuda")
    foff0 = encode(torch, codec, level, d_in, n, chunk, d_cb, nch, work0, out0)
    framed0 = out0[: int(foff0[-1])].clone()
    del work0, out0

    work = torch.full((wb + GUARD,), 0xA5, dtype=torch.uint8, device="cuda")
    out = torch.full((ob + GUARD,), 0x5A, dtype=torch.uint8, device="cuda")
    foff = encode(torch, codec, level, d_in, n, chunk, d_cb, nch, work, out)
    assert bool((work[wb:] == 0xA5).all()), "the encoder wrote past its workspace"
    assert bool((out[ob:] == 0x5A).all()), "the encoder wrote past the output bound"
    assert torch.equal(foff, foff0)
    assert torch.equal(out[: int(foff[-1])], framed0), "the frames depend on what the workspace held"
