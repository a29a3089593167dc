"""GPU tests of zmt_zstd_compress_dict_device: every stream equals the CPU twin's (_zdictenc.framed_b200) byte for byte,
and every frame is restored by libzstd's ZSTD_decompress_usingDict and by the GPU decoder against the same dictionary
(host scan, container index and plain index).  Also: dictionary buffers at every address mod 16, a batch over two chunk
groups, incompressible records within zmt_zstdc_out_bound, the calls that must equal the call without a dictionary
(NULL index, empty raw content, an index built on a failed load) and the levels the call refuses."""
import ctypes

import numpy as np
import pytest
import torch

import zstdmt_b200 as z
import _zdict as zd
import _zdictenc as zde
import test_gpu_zstd_dict as gd

pytestmark = pytest.mark.gpu

GROUP_BYTES = 256 << 20                  # ZL_GROUP_BYTES


def slots(recs, chunk):
    src = np.zeros(len(recs) * chunk, np.uint8)
    for i, r in enumerate(recs):
        src[i * chunk: i * chunk + r.size] = r
    return src, np.array([r.size for r in recs], np.uint32)


def gpu_stream(src, chunk, level, dct=None, cb=None):
    comp = z.ZstdDeviceCompressor(src.size, chunk, level=level, dictionary=dct)
    d_cb = torch.from_numpy(cb.astype(np.int32)).cuda() if cb is not None else None
    if cb is not None:
        assert comp.nchunks == cb.size
    out, foff = comp.run(torch.from_numpy(src).cuda(), chunk_bytes=d_cb)
    torch.cuda.synchronize()
    return out[: int(foff[-1].item())].cpu().numpy(), comp


def check_twin(got, src, chunk, level, D, did, cb=None):
    want = zde.framed_b200(src, chunk, level, cb, D, did)
    assert got.size == want.size and np.array_equal(got, want), "level %d: GPU stream differs from the twin" % level


def record_batch(seed, n):
    return zd.records(seed, n, lo=1024, hi=4096)


@pytest.fixture(scope="module")
def trained():
    d = zd.train(7, 32 << 10)
    return d, z.ZstdDictionary(d)


@pytest.mark.parametrize("level", [6, 9, 12, 19])
def test_streams_equal_the_twin_and_decode(trained, level):
    d, dct = trained
    D, did = zde.content(d), zd.dict_id(d)
    recs = record_batch(level, 48)
    src, cb = slots(recs, 4096)                               # explicit sizes: records in 4 KiB slots
    got, _ = gpu_stream(src, 4096, level, dct, cb)
    check_twin(got, src, 4096, level, D, did, cb)
    gd.check(zde.frames(got), recs, d, dct, seed=level)
    txt = np.concatenate(record_batch(level + 100, 60))      # implicit sizes: one input cut every 64 KiB
    got, _ = gpu_stream(txt, 65536, level, dct)
    check_twin(got, txt, 65536, level, D, did)
    gd.check(zde.frames(got), [txt[i: i + 65536] for i in range(0, txt.size, 65536)], d, dct, seed=level + 1)


@pytest.mark.parametrize("dict_id", [0, 7, 300, 70000])
def test_dictionary_ids_and_raw_content(dict_id):
    content = np.concatenate(zd.records(32, 60))[: 24 << 10]
    d = content if dict_id == 0 else zd.finalize(9, content, 32 << 10, level=9, dict_id=dict_id)
    dct = z.ZstdDictionary(d)
    recs = record_batch(dict_id + 3, 24)
    src, cb = slots(recs, 4096)
    got, _ = gpu_stream(src, 4096, 9, dct, cb)
    check_twin(got, src, 4096, 9, zde.content(d), zd.dict_id(d), cb)
    gd.check(zde.frames(got), recs, d, dct)


def raw_api_stream(src, chunk, level, d_cdict, cb=None):
    L = z.lib()
    n = L.zmt_chunk_count(src.size, chunk) if cb is None else cb.size
    work = torch.empty(L.zmt_zstdc_level_workspace_bytes(n, chunk, level), dtype=torch.uint8, device="cuda")
    out = torch.empty(L.zmt_zstdc_out_bound(n, chunk), dtype=torch.uint8, device="cuda")
    foff = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    d_in = torch.from_numpy(src).cuda()
    d_cb = torch.from_numpy(cb.astype(np.int32)).cuda() if cb is not None else None
    rc = L.zmt_zstd_compress_dict_device(d_in.data_ptr(), src.size, chunk, d_cb.data_ptr() if cb is not None else None, n, level,
                                         work.data_ptr(), out.data_ptr(), foff.data_ptr(), torch.cuda.current_stream().cuda_stream, d_cdict)
    assert rc == 0, z.ST_NAMES.get(rc, rc)
    torch.cuda.synchronize()
    return out[: int(foff[-1].item())].cpu().numpy()


def load_at(d, shift):
    """Load d from a device buffer placed at `shift` bytes past a 256-byte boundary and build its index there: (ddict
    record, info, index, the buffers they point into)."""
    L = z.lib()
    buf = torch.zeros(d.size + 64, dtype=torch.uint8, device="cuda")
    buf[shift: shift + d.size] = torch.from_numpy(d).cuda()
    dd = torch.zeros(L.zmt_zstd_ddict_bytes(), dtype=torch.uint8, device="cuda")
    info = torch.zeros(ctypes.sizeof(z.DictInfo), dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    assert L.zmt_zstd_ddict_load_device(buf.data_ptr() + shift, d.size, dd.data_ptr(), info.data_ptr(), st) == 0
    cd = torch.empty(L.zmt_zstd_cdict_bytes(d.size), dtype=torch.uint8, device="cuda")
    assert L.zmt_zstd_cdict_build_device(dd.data_ptr(), d.size, cd.data_ptr(), st) == 0
    torch.cuda.synchronize()
    return dd, z.DictInfo.from_buffer_copy(info.cpu().numpy().tobytes()), cd, buf


def test_dictionary_at_every_address_mod_16(trained):
    d, _ = trained
    recs = record_batch(77, 16)
    src, cb = slots(recs, 4096)
    want = zde.framed_b200(src, 4096, 9, cb, zde.content(d), zd.dict_id(d))
    raw = np.concatenate(zd.records(78, 30))[: 9999]
    want_raw = zde.framed_b200(src, 4096, 9, cb, raw, 0)
    for shift in range(16):
        for dd_, w in ((d, want), (raw, want_raw)):
            _, info, cd, _ = load_at(dd_, shift)
            assert info.status == 0
            assert np.array_equal(raw_api_stream(src, 4096, 9, cd.data_ptr(), cb), w), shift


def test_batch_over_two_chunk_groups(trained):
    d, dct = trained
    chunk = 96 << 20                                          # two chunks per group: three chunks are two groups
    assert GROUP_BYTES // chunk == 2
    recs = record_batch(91, 3)
    src, cb = slots(recs, chunk)
    for level in (6, 12):
        got, _ = gpu_stream(src, chunk, level, dct, cb)
        check_twin(got, src, chunk, level, zde.content(d), zd.dict_id(d), cb)


def test_incompressible_records_fit_the_bound(trained):
    d, dct = trained
    rng = np.random.default_rng(5)
    recs = [rng.integers(0, 256, int(n)).astype(np.uint8) for n in rng.integers(1, 4097, 64)]
    src, cb = slots(recs, 4096)
    got, comp = gpu_stream(src, 4096, 12, dct, cb)
    assert got.size <= z.lib().zmt_zstdc_out_bound(comp.nchunks, 4096)
    check_twin(got, src, 4096, 12, zde.content(d), zd.dict_id(d), cb)
    gd.check(zde.frames(got), recs, d, dct)


def test_calls_equal_to_the_call_without_a_dictionary():
    L = z.lib()
    recs = record_batch(55, 24)
    src, cb = slots(recs, 4096)
    for level in (6, 12):
        plain, _ = gpu_stream(src, 4096, level, None, cb)
        assert np.array_equal(raw_api_stream(src, 4096, level, None, cb), plain)            # d_cdict = NULL
        empty = z.ZstdDictionary(b"")
        assert empty.info.status == 0 and empty.info.content_bytes == 0
        got, _ = gpu_stream(src, 4096, level, empty, cb)
        assert np.array_equal(got, plain)
        bad = np.concatenate([np.array([zd.DICT_MAGIC, 1234], "<u4").view(np.uint8), np.full(200, 0xFF, np.uint8)])
        _, info, cd, _ = load_at(bad, 0)                     # a formatted dictionary whose tables the load refuses
        assert info.status != 0
        assert np.array_equal(raw_api_stream(src, 4096, level, cd.data_ptr(), cb), plain)
    assert L.zmt_zstd_cdict_bytes(1 << 31) == 0


def test_levels_below_6_are_refused(trained):
    _, dct = trained
    L = z.lib()
    src = np.zeros(4096, np.uint8)
    d_in = torch.from_numpy(src).cuda()
    work = torch.empty(L.zmt_zstdc_level_workspace_bytes(1, 4096, 6), dtype=torch.uint8, device="cuda")
    out = torch.empty(L.zmt_zstdc_out_bound(1, 4096), dtype=torch.uint8, device="cuda")
    foff = torch.zeros(2, dtype=torch.int64, device="cuda")
    for level in range(1, 6):
        rc = L.zmt_zstd_compress_dict_device(d_in.data_ptr(), 4096, 4096, None, 1, level, work.data_ptr(), out.data_ptr(), foff.data_ptr(),
                                             torch.cuda.current_stream().cuda_stream, dct.cdict().data_ptr())
        assert rc == 12                                       # ZMT_ST_BAD_ARG
        with pytest.raises(ValueError):
            z.ZstdDeviceCompressor(4096, 4096, level=level, dictionary=dct)
