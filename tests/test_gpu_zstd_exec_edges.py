"""The GPU zstd decoder on the x_* cases of _zcorpus.py, which put the execute pass (zx_block) and the lane sequence
reader at the edges of their schedules (tests/_zxmodel.py names the edges; test_zstd_exec_model.py asserts that each case
reaches them): all cases in one batch with frame i at input address i mod 8 (every alignment of the lane reader's loads),
the same batch through the device-built block table, and each case side by side with frames the lane decoder hands to
the general path."""
import ctypes

import numpy as np
import pytest

import _zcorpus as zc
import zstdmt_b200 as z
from test_gpu_zstd_decode_edges import check_outputs, device_decode, framed
from test_zstd_decode_corpus import ZF_NEEDS_SEQ

pytestmark = pytest.mark.gpu
X_CASES = list(zc.X_CASES)


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def padded_decoder(torch, frames):
    """A ZstdDeviceDecompressor over the frames with frame i (its zstd magic) at input address i mod 8: pad bytes go
    between the container frames, and the block table is built with zmt_zstd_scan_frame_host at each frame's absolute
    offset.  Returns (decoder, device input)."""
    L = z.lib()
    parts, offs, pos = [], [], 0
    for i, f in enumerate(frames):
        pad = (i - (pos + 12)) % 8
        parts += [np.zeros(pad, np.uint8), framed([f])]
        pos += pad
        offs.append(pos + 12); pos += 12 + f.size
    fb = np.concatenate(parts)
    assert [o % 8 for o in offs] == [i % 8 for i in range(len(frames))]
    n, dsz = len(frames), L.zmt_zstd_blk_desc_bytes()
    cap = fb.size // 3 + n + 16
    blocks = np.zeros(cap * dsz, np.uint8)
    nblk, scr = ctypes.c_uint32(0), ctypes.c_uint64(0)
    first, expect, fseq = np.zeros(n + 1, np.int32), np.zeros(n, np.int64), np.zeros(n, np.int32)
    for i, (o, f) in enumerate(zip(offs, frames)):
        first[i] = nblk.value
        cs, fl = ctypes.c_uint64(0), ctypes.c_uint32(0)
        rc = L.zmt_zstd_scan_frame_host(fb[o:].ctypes.data, f.size, o, i, blocks.ctypes.data, ctypes.byref(nblk), cap,
                                        ctypes.byref(scr), ctypes.byref(cs), ctypes.byref(fl))
        assert rc == 0, (i, rc)
        expect[i], fseq[i] = cs.value, fl.value
    first[n] = nblk.value
    dec = z.ZstdDeviceDecompressor.__new__(z.ZstdDeviceDecompressor)
    dec.n, dec.nblk = n, nblk.value
    oo = np.zeros(n + 1, np.int64); oo[1:] = np.cumsum(expect)
    dec.out_total = int(oo[-1])
    dev = "cuda"
    dec.d_blocks = torch.from_numpy(blocks[: max(1, dec.nblk) * dsz].copy()).to(dev)
    dec.d_first, dec.d_expect = torch.from_numpy(first).to(dev), torch.from_numpy(expect).to(dev)
    dec.d_fseq, dec.d_out_off = torch.from_numpy(fseq).to(dev), torch.from_numpy(oo).to(dev)
    dec.out = torch.empty(max(dec.out_total, 1), dtype=torch.uint8, device=dev)
    dec.out_size = torch.zeros(n, dtype=torch.int64, device=dev)
    dec.status = torch.zeros(n, dtype=torch.int32, device=dev)
    dec.work = torch.empty(L.zmt_zstdd_workspace_bytes(n, dec.nblk, scr.value), dtype=torch.uint8, device=dev)
    return dec, torch.from_numpy(fb).to(dev)


def expect_route(name, fseq):
    """Level-1 cases and x_budget take the lane decoder (no flag), level-19 cases the dependent-block route."""
    if name.endswith("_l19"):
        assert fseq & ZF_NEEDS_SEQ, name
    else:
        assert not fseq & ZF_NEEDS_SEQ, name


def test_gpu_decodes_x_cases_at_every_input_alignment(gpu):
    """All x_* cases in one batch, twice over, so that frame i starts at input address i mod 8 for every case at two
    residues: status 0, the content size, the source bit for bit; the routes as the traces show them."""
    names = X_CASES + X_CASES[::-1]
    srcs, frames = zip(*(zc.case(n) for n in names))
    dec, d_in = padded_decoder(gpu, list(frames))
    out, st = dec.run(d_in)
    gpu.cuda.synchronize()
    check_outputs(out.cpu().numpy(), st.cpu().numpy(), dec.out_size.cpu().numpy(), list(srcs))
    fseq = dec.d_fseq.cpu().numpy()
    for i, n in enumerate(names):
        expect_route(n, int(fseq[i]))


def test_gpu_decodes_x_cases_through_device_block_table(gpu):
    """The same cases in one batch through ZstdDeviceDecompressor.from_device (frame index and block table built on the
    GPU)."""
    srcs, frames = zip(*(zc.case(n) for n in X_CASES))
    d_in = gpu.from_numpy(framed(list(frames))).cuda()
    dec = z.ZstdDeviceDecompressor.from_device(d_in)
    assert dec.n == len(X_CASES)
    out, st = dec.run(d_in)
    gpu.cuda.synchronize()
    check_outputs(out.cpu().numpy(), st.cpu().numpy(), dec.out_size.cpu().numpy(), list(srcs))


@pytest.mark.parametrize("name", X_CASES)
def test_gpu_decodes_x_case_among_fallback_frames(gpu, name):
    """Each case between frames whose blocks the lane decoder hands on (offset codes above 24; repeat offsets found at
    run time), so that lane-route and fallback blocks share the decoder's warps."""
    names = ["reps_predef", name, "far_predef", name, "reps_predef"]
    srcs, frames = zip(*(zc.case(n) for n in names))
    dec, out, st, sz = device_decode(gpu, list(frames))
    check_outputs(out, st, sz, list(srcs))
    expect_route(name, int(dec.d_fseq.cpu().numpy()[1]))
