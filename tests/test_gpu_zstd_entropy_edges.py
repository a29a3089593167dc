"""The zstd encoder's entropy stage (z_encode_block) on the GPU at the edges the corpus of _zentcorpus reaches
(pytest -m gpu): every case's input is compressed at level 3, and at level 9 when the case was built for that level,
and the framed stream must equal the CPU twin's (_zenc.framed_b200) byte for byte.  The checks of
test_gpu_zstd_encoder.check / test_gpu_zstd_levels.check run too: parse, sub-block cut, Huffman code, mode rules and the
round trip through the oracle, libzstd and the GPU decoder.  Which edge each case reaches, and that its knock-out does
not, is checked on the CPU (test_zstd_enc_twin.py)."""
import numpy as np
import pytest

import _zentcorpus as zc
import test_gpu_zstd_encoder as t3
import test_gpu_zstd_levels as t9

pytestmark = pytest.mark.gpu
CASES = {c.name: c for c in zc.cases()}


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch


@pytest.mark.parametrize("name", sorted(CASES))
def test_entropy_edge_is_byte_identical_to_the_twin(torch, name):
    c = CASES[name]
    src, chunk, cb = c.built()
    t3.check(torch, src, chunk, cb)
    if c.level != 3:
        t9.check(torch, src, chunk, c.level, cb)


def test_knocked_out_inputs_are_byte_identical_too(torch):
    """The knock-out inputs, all of them through level 3 in one stream of explicit chunk sizes."""
    parts = [CASES[n].knocked()[0] for n in sorted(CASES)]
    parts = [p for p in parts if p.size <= 1 << 20]
    chunk = max(p.size for p in parts)
    src = np.zeros(chunk * len(parts), np.uint8)
    for i, p in enumerate(parts):
        src[i * chunk: i * chunk + p.size] = p
    t3.check(torch, src, chunk, [p.size for p in parts])
