"""The decoders' workspace sizes (CPU).  zmt_lz4d_workspace_bytes keeps the size rule it has always had;
zmt_zstdd_workspace_bytes keeps its rule less one region of a256(8 * nframes) that the launcher never used.  Both rules
are restated here from before their layouts moved into lz4d_layout (lz4_kernels.cu) and zstdd_layout (zstd_decode.cu).
The index and range-read sizes ask cub for its scan storage and need a device: tests/test_gpu_decoder_workspace.py."""
import itertools

import pytest

import zstdmt_b200 as z

LZBLK_BYTES = 20                    # sizeof(LzBlk), lz4_decode.cuh: five uint32_t
TICKET_WIN = 16384                  # MX_TICKET_WIN, match_exec.cuh
COUNTS = [0, 1, 2, 255, 256, 257, 10 ** 6]
IN_BYTES = [0, 1, 2, 3, (1 << 32) + 5]
SCRATCH = [0, 1, 4096]


def a256(x):
    return (x + 255) & ~255


def ticket_table(nframes):
    return a256((nframes // TICKET_WIN + 2) * 8)


@pytest.mark.parametrize("nframes", COUNTS)
def test_lz4_decoder_workspace_bytes(nframes):
    L = z.lib()
    nf = nframes
    for ns, n in itertools.product(COUNTS, IN_BYTES):
        want = (3 * a256(nf * 4) + 256 + 2 * a256((nf + 1) * 8) + ticket_table(nf) + a256(ns * LZBLK_BYTES) + a256(ns * 4)
                + a256((n // 3 + 8) * 8) + 1024)
        assert L.zmt_lz4d_workspace_bytes(nf, ns, n) == want, (nf, ns, n)


@pytest.mark.parametrize("nframes", COUNTS)
def test_zstd_decoder_workspace_bytes(nframes):
    L = z.lib()
    nf = nframes
    for nb, s in itertools.product(COUNTS, SCRATCH):
        before = a256(nb * 4) * 2 + a256(nb * 8) + a256(nf * 8) + 256 + ticket_table(nf) + 3 * a256(nb * 4) + s + 1024
        assert L.zmt_zstdd_workspace_bytes(nf, nb, s) == before - a256(8 * nf), (nf, nb, s)
