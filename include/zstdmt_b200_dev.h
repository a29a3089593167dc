/* zstdmt_b200_dev.h — device-resident batch entry points of libzstdmt_b200.so.
 *
 * These are what the host pipeline behind LZ4MT_* / ZSTDCB_* calls per batch, exported so a
 * caller that already holds its data in HBM (bench.py's device-timed metric, a GPU-side
 * producer) can skip the host staging.  Plain C ABI: device pointers + sizes + a CUDA stream
 * handle passed as void*.  All work is enqueued on `stream`; nothing synchronises.
 *
 * What each call replaces in the reference (one call = the codec step of every worker
 * iteration of a whole batch of chunks):
 *   zmt_lz4_compress_device    LZ4F_compressFrame + 12-byte header, lib/lz4-mt_compress.c:280-298
 *                              (zmt_lz4_compress_level_device: the same at a level)
 *   zmt_lz4_decompress_device  LZ4F_decompress, lib/lz4-mt_decompress.c:328-362
 *   zmt_zstd_compress_device   ZSTD_compress + 12-byte header, lib/zstd-mt_compress.c:284-302
 *   zmt_zstd_decompress_device ZSTD_decompressStream loop, lib/zstd-mt_decompress.c:442-527
 */
#ifndef ZSTDMT_B200_DEV_H
#define ZSTDMT_B200_DEV_H
#include <stddef.h>
#include <stdint.h>

#define ZMT_LZ4_TMP_STRIDE 65824u     /* >= LZ4 worst case for a 64 KiB block (65536 + 257 + 16), 16-byte multiple */

/* per-frame / per-call status codes */
#define ZMT_ST_OK               0u
#define ZMT_ST_TRUNCATED        1u
#define ZMT_ST_BAD_MAGIC        2u
#define ZMT_ST_BAD_HEADER       3u
#define ZMT_ST_HDR_CHECKSUM     4u
#define ZMT_ST_BLOCK            5u
#define ZMT_ST_DST_SMALL        6u
#define ZMT_ST_CONTENT_CHECKSUM 7u
#define ZMT_ST_CONTENT_SIZE     8u
#define ZMT_ST_TRAILING         9u
#define ZMT_ST_UNSUPPORTED      10u
#define ZMT_ST_CUDA             11u
#define ZMT_ST_BAD_ARG          12u
#define ZMT_ST_DICT_WRONG       13u      /* the frame names a Dictionary_ID other than the dictionary given */
#define ZMT_ST_HAS_CHK          0x100u   /* internal flag between decode and verify kernels */

#ifdef __cplusplus
extern "C" {
#endif

/* number of chunks (= frames) an input of in_bytes cut every chunk_size bytes produces;
 * an empty input still yields one frame (lib/lz4-mt_compress.c:265) */
uint32_t zmt_chunk_count(uint64_t in_bytes, uint32_t chunk_size);

/* ---- LZ4 ----
 * Input layout: chunk c starts at d_in + c*chunk_size.  Its length is d_chunk_bytes[c] when
 * that (device) array is given, else derived from in_bytes (all full, last one short).
 * Output: the framed stream, frames back to back; d_frame_off[c] = offset of frame c's
 * 12-byte skippable header, d_frame_off[nchunks] = total bytes. */
size_t   zmt_lz4c_workspace_bytes(uint32_t nchunks, uint32_t chunk_size);
uint64_t zmt_lz4c_out_bound(uint32_t nchunks, uint32_t chunk_size);
int      zmt_lz4_compress_device(const void* d_in, uint64_t in_bytes, uint32_t chunk_size, const uint32_t* d_chunk_bytes,
                                 uint32_t nchunks, void* d_work, void* d_out, uint64_t* d_frame_off, void* stream);
/* The same at an LZ4 level.  Levels 1-9 run the encoder above (same bytes, same workspace: independent blocks, FLG 0x6C).
 * Levels 10-12 run the high-compression class: hash chains over the whole chunk walked to a per-level depth, a lazy
 * parse, and linked 64 KiB blocks (FLG 0x4C, 0x44 for an empty chunk) whose matches may reach up to 65535 bytes back
 * into the chunk's earlier blocks.  Any other level returns ZMT_ST_BAD_ARG (the workspace size is then 0).  The
 * workspace depends on the level; out_bound does not. */
size_t   zmt_lz4c_level_workspace_bytes(uint32_t nchunks, uint32_t chunk_size, int level);
int      zmt_lz4_compress_level_device(const void* d_in, uint64_t in_bytes, uint32_t chunk_size, const uint32_t* d_chunk_bytes,
                                       uint32_t nchunks, int level, void* d_work, void* d_out, uint64_t* d_frame_off, void* stream);

/* d_in/in_bytes = the framed stream in HBM; d_frame_off[f] = offset of frame f's 12-byte header, d_frame_csize[f] =
 * its payload size; d_out_off[f..f+1] = where frame f's content goes and how much room it has;
 * nslots = sum over frames of max(1, ceil(room_f / 64 KiB)): the capacity of the block table (one warp per LZ4F block,
 * two passes: token parse + literals, then match execution; frames with linked blocks — what liblz4 emits for the
 * reference — decode block-parallel too, a block waits on the previous one only where a match reaches into it);
 * d_out_size[f] / d_status[f] receive decoded bytes and a ZMT_ST_* code. */
size_t   zmt_lz4d_workspace_bytes(uint32_t nframes, uint32_t nslots, uint64_t in_bytes);
int      zmt_lz4_decompress_device(const void* d_in, uint64_t in_bytes, const uint64_t* d_frame_off, const uint32_t* d_frame_csize, uint32_t nframes,
                                   uint32_t nslots, void* d_out, const uint64_t* d_out_off, uint64_t* d_out_size,
                                   uint32_t* d_status, void* d_work, void* stream);

/* ---- Zstandard ----  same layout contract as the LZ4 entry points; frames are single-segment zstd frames
 * (magic, FHD, content size, blocks, no checksum) behind the same 12-byte container header. */
size_t   zmt_zstdc_workspace_bytes(uint32_t nchunks, uint32_t chunk_size);
uint64_t zmt_zstdc_out_bound(uint32_t nchunks, uint32_t chunk_size);
int      zmt_zstd_compress_device(const void* d_in, uint64_t in_bytes, uint32_t chunk_size, const uint32_t* d_chunk_bytes,
                                  uint32_t nchunks, void* d_work, void* d_out, uint64_t* d_frame_off, void* stream);
/* The same at a zstd level.  Levels 1-5 run the level-3 encoder above (same bytes, same workspace).  Levels 6-12 run
 * the search class with chunk-wide hash chains and a lazy parse, each level with its own parameters; 13-22 use
 * level 12's.  Its match window is 2 MiB (levels 6-9) or 4 MiB (10 and up), offsets may reach the whole chunk's
 * history within that window, blocks are 16 KiB.  The workspace depends on the level; out_bound does not. */
size_t   zmt_zstdc_level_workspace_bytes(uint32_t nchunks, uint32_t chunk_size, int level);
int      zmt_zstd_compress_level_device(const void* d_in, uint64_t in_bytes, uint32_t chunk_size, const uint32_t* d_chunk_bytes,
                                        uint32_t nchunks, int level, void* d_work, void* d_out, uint64_t* d_frame_off, void* stream);

/* Decode.  The host walks frame + block headers (3 bytes per block, plus the two section headers of compressed
 * blocks) with zmt_zstd_scan_frame_host — exactly what the pipeline's reader thread does while it parses frames —
 * and hands the device a block table: one warp per block for entropy decoding, a scan for the output offsets, one
 * warp per block for sequence execution.  Descriptors are opaque (zmt_zstd_blk_desc_bytes() each). */
size_t   zmt_zstd_blk_desc_bytes(void);
int      zmt_zstd_scan_frame_host(const uint8_t* frame, size_t n, uint64_t base_off, uint32_t frame_idx, void* blocks_out,
                                  uint32_t* nblocks_io, uint32_t max_blocks, uint64_t* scratch_used, uint64_t* content_size,
                                  uint32_t* needs_seq /* 1: blocks depend on earlier ones -> frame-sequential entropy pass */);
size_t   zmt_zstdd_workspace_bytes(uint32_t nframes, uint32_t nblocks, uint64_t scratch_bytes);
int      zmt_zstd_decompress_device(const void* d_in, const void* d_blocks, uint32_t nblocks, const uint32_t* d_frame_first_blk,
                                    const uint64_t* d_expect, const uint32_t* d_frame_seq, uint32_t nframes, void* d_out,
                                    const uint64_t* d_out_off, uint64_t* d_out_size, uint32_t* d_status, void* d_work, void* stream);

/* ---- Frame index on the device: the tables of the two decode calls above, built on the GPU from a container-framed
 * stream ([LE32 0x184D2A50][LE32 4][LE32 size] + payload, repeated) that is already in HBM, for callers whose stream
 * arrives there without passing the host (GPUDirect Storage, NCCL, the device compressors).  The host reads back only
 * the zmt_frame_index summary to size its allocations; the tables are exactly the arguments the decode calls take.
 *
 *   zmt_lz4_index_device   fills d_frame_off[f], d_frame_csize[f] (f < min(nframes, max_frames)) and d_out_off[0..max_frames]:
 *                          frame f's room is its LZ4F content size, or the block bound without one, as the host pipeline
 *                          gives it; info.nblocks = the nslots argument of zmt_lz4_decompress_device.
 *   zmt_zstd_index_device  fills the same three plus d_frame_first_blk[0..max_frames], d_frame_scratch[0..max_frames] (scratch
 *                          base of each frame's blocks), d_expect[f] (content size, ~0 for a frame without one: its room is
 *                          the block bound) and d_frame_seq[f] (ZF_* flags); info.nblocks descriptors and info.scratch_bytes
 *                          (the third argument of zmt_zstdd_workspace_bytes) are what to allocate.
 *   zmt_zstd_blocks_device then writes the info.nblocks descriptors into d_blocks, byte for byte what zmt_zstd_scan_frame_host
 *                          writes for the same frames.
 * Arrays indexed 0..max_frames hold max_frames + 1 entries; entry nframes is the total.  d_work: zmt_index_workspace_bytes.
 * Streams up to 3 * (2^32 - 1) bytes (ZMT_ST_BAD_ARG above).  Every read stays inside [d_in, d_in + in_bytes).
 *
 * info.status, each the decision the host pipeline takes on the same bytes; the first failure in stream order wins:
 *   ZMT_ST_BAD_MAGIC    a container header with the wrong magic, or a length field other than 4 (bad_frame = nframes)
 *   ZMT_ST_TRUNCATED    a container header or payload runs past in_bytes (bad_frame = nframes)
 *   ZMT_ST_BAD_HEADER   LZ4: an unusable LZ4F header, or a content size above 255 * payload + 65536 (bad_offset = the payload)
 *                       An LZ4 payload without the LZ4F magic gets room 0 and indexes fine; the decoder reports BAD_MAGIC.
 *   zstd: what zmt_zstd_scan_frame_host returns for the frame (BAD_MAGIC, BAD_HEADER, UNSUPPORTED for a dictionary ID,
 *                       BLOCK, TRUNCATED, TRAILING; with a dictionary DICT_WRONG, bad_offset = the frame's start); bad_offset = the frame or block header the walk stopped at, or the
 *                       first trailing byte
 *   ZMT_ST_DST_SMALL    more than max_frames frames: nframes is the true count, bad_frame = max_frames, bad_offset its header
 *   in_bytes == 0       ZMT_ST_OK with nframes = 0
 * With ZMT_ST_OK, bad_frame = nframes and bad_offset = 0.  The other fields are only meaningful with ZMT_ST_OK.
 * The calls return ZMT_ST_OK once enqueued, ZMT_ST_BAD_ARG or ZMT_ST_CUDA. */
typedef struct {
    uint32_t status;        /* ZMT_ST_OK or the first failure met */
    uint32_t bad_frame;     /* frame it was met in (== nframes when the container itself is at fault) */
    uint64_t bad_offset;    /* stream offset where the walk stopped */
    uint32_t nframes;       /* frames in the stream, also when > max_frames (status ZMT_ST_DST_SMALL) */
    uint32_t nblocks;       /* zstd: descriptors to allocate; lz4: block-table slots (the nslots argument) */
    uint64_t out_bytes;     /* d_out_off[nframes] */
    uint64_t scratch_bytes; /* zstd: third argument of zmt_zstdd_workspace_bytes */
} zmt_frame_index;

size_t zmt_index_workspace_bytes(uint32_t max_frames);
int    zmt_lz4_index_device(const void* d_in, uint64_t in_bytes, uint32_t max_frames, uint64_t* d_frame_off, uint32_t* d_frame_csize,
                            uint64_t* d_out_off, zmt_frame_index* d_info, void* d_work, void* stream);
int    zmt_zstd_index_device(const void* d_in, uint64_t in_bytes, uint32_t max_frames, uint64_t* d_frame_off, uint32_t* d_frame_csize,
                             uint32_t* d_frame_first_blk, uint64_t* d_frame_scratch, uint64_t* d_expect, uint32_t* d_frame_seq,
                             uint64_t* d_out_off, zmt_frame_index* d_info, void* d_work, void* stream);
int    zmt_zstd_blocks_device(const void* d_in, uint32_t nframes, const uint64_t* d_frame_off, const uint32_t* d_frame_csize,
                              const uint32_t* d_frame_first_blk, const uint64_t* d_frame_scratch, void* d_blocks, uint32_t nblocks, void* stream);

/* ---- Frame index on the device for plain streams: the same tables and summary from an ordinary .lz4 / .zst file in
 * HBM (codec frames back to back as the lz4 and zstd tools write them, without container headers; skippable frames,
 * magic 0x184D2A50..0x184D2A5F + LE32 size + payload, anywhere between them).  Arguments, workspace, max_frames and
 * ZMT_ST_DST_SMALL as for the container calls above.  One thread walks the stream: a frame's end is only known by
 * walking its block headers (one dependent load per block header).  Each frame start is decided as the callback API's
 * plain path decides it on the same bytes.  Skippable frames are not frames of the index: nframes counts codec frames,
 * so a container-framed stream is also a valid plain stream, each 12-byte header a skippable frame of size 4.
 *
 * Layout convention.  The tables are written for a base 12 bytes below the stream, so that the decode calls address a
 * frame as they address one behind a container header: d_frame_off[f] = frame f's offset in the plain stream,
 * d_frame_csize[f] = its length, and the zstd descriptors' offsets are relative to d_in - 12.  Call
 * zmt_zstd_blocks_device, zmt_lz4_decompress_device (with in_bytes + 12) and zmt_zstd_decompress_device unchanged with
 * d_in - 12.  None of them reads below base + 12, where the stream starts: every read is at
 * base + frame_off + 12 or a descriptor's offset on, apart from aligned 8- and 16-byte loads of the decoders, whose
 * aligned word always holds a stream byte and so never leaves the caller's allocation.
 *
 * info.status, the plain path's decision at the first frame start that fails (the walk ends there: the next frame's
 * start is not known behind it); bad_frame = the frames accepted before it, bad_offset in stream coordinates:
 *   ZMT_ST_TRUNCATED    fewer than 4 bytes at a frame start, or a skippable frame whose size runs past the end; an LZ4F
 *                       header shorter than 7 bytes (the frame's start) / LZ4F: the header or a block runs past the end
 *                       (the block header the walk could not read, or in_bytes)
 *   ZMT_ST_BAD_MAGIC    neither a skippable frame nor the codec's magic, zstd legacy magics included (the frame's start)
 *   ZMT_ST_BAD_HEADER   LZ4F: FLG version other than 01, or a block-size id below 4 (the frame's start)
 *   ZMT_ST_CONTENT_SIZE LZ4F: a content size above the bound of its blocks (the frame's start)
 *   zstd: what zmt_zstd_scan_frame_host returns for the frame (BAD_HEADER, UNSUPPORTED for a dictionary ID, BLOCK,
 *                       TRUNCATED), bad_offset = the header element the walk stopped at
 *   ZMT_ST_UNSUPPORTED  a frame of 2^32 bytes or more (the frame's start): the decode calls' frame_csize is 32-bit; the
 *                       callback API decodes such a frame in segments
 *   ZMT_ST_DST_SMALL    as above
 * ZMT_ST_TRAILING cannot occur: bytes behind a frame are the next frame.  An empty stream, or one of skippable frames
 * only, is ZMT_ST_OK with nframes = 0. */
int    zmt_lz4_index_plain_device(const void* d_in, uint64_t in_bytes, uint32_t max_frames, uint64_t* d_frame_off, uint32_t* d_frame_csize,
                                  uint64_t* d_out_off, zmt_frame_index* d_info, void* d_work, void* stream);
int    zmt_zstd_index_plain_device(const void* d_in, uint64_t in_bytes, uint32_t max_frames, uint64_t* d_frame_off, uint32_t* d_frame_csize,
                                   uint32_t* d_frame_first_blk, uint64_t* d_frame_scratch, uint64_t* d_expect, uint32_t* d_frame_seq,
                                   uint64_t* d_out_off, zmt_frame_index* d_info, void* d_work, void* stream);

/* ---- zstd frames written with a dictionary (RFC 8878 §5) ----
 * A dictionary is loaded once on the device and then named by the calls below, which are the calls above plus the
 * record.  Two kinds are accepted, as libzstd's ZSTD_dct_auto accepts them:
 *   formatted    magic 0xEC30A437, LE32 Dictionary_ID, the entropy tables (a Huffman tree description in the literals
 *                section's format, then FSE table descriptions for OF, ML and LL, in that order), three LE32 repeat
 *                offsets (each non-zero and at most the content size), then the content: the rest of the buffer;
 *   raw content  any other buffer: Dictionary_ID 0, no tables, repeat offsets {1, 4, 8}, all of it content.
 * zmt_zstd_ddict_load_device parses and checks the entropy section with one warp, using the decoder's own table
 * builders and the block format's limits (Huffman codes up to 11 bits, FSE logs 8 for OF and 9 for ML / LL), and writes
 * the opaque record d_ddict (zmt_zstd_ddict_bytes() bytes of device memory) and the summary d_info.  The record keeps
 * the address d_dict: the dictionary bytes stay where the caller put them and must outlive every call that names the
 * record.  No per-frame memory: the frames read the content in place.  d_info->status: ZMT_ST_OK, ZMT_ST_BAD_HEADER
 * (unusable tables or repeat offsets), ZMT_ST_TRUNCATED (fewer than 12 bytes behind the tables for the repeat offsets);
 * a record whose load failed makes every frame named against it fail with that status.  Reports under
 * ZMT_K_ZSTD_DECODE; returns ZMT_ST_OK once enqueued, ZMT_ST_BAD_ARG or ZMT_ST_CUDA.
 *
 * The rule is libzstd's ZSTD_decompress_usingDict: every frame of a dictionary batch decodes against the dictionary,
 * whether its header names the dictionary's ID or names none.  A frame that names another ID fails with
 * ZMT_ST_DICT_WRONG (the index's bad_offset: the frame's start).  Each frame gets ZF_DICT | ZF_NEEDS_SEQ in d_frame_seq:
 * the tables and repeat offsets its first blocks may take from the dictionary tie it to the dependent-block route.
 * Matches may reach as far back as the frame's output so far plus the dictionary's content.
 *   zmt_zstd_scan_frame_dict_host       zmt_zstd_scan_frame_host with the summary of a loaded dictionary (dict = NULL:
 *                                       no dictionary, which is zmt_zstd_scan_frame_host itself)
 *   zmt_zstd_index_dict_device,         the index calls; d_ddict = NULL is the call without a dictionary
 *   zmt_zstd_index_plain_dict_device
 *   zmt_zstd_blocks_dict_device         zmt_zstd_blocks_device; byte for byte what zmt_zstd_scan_frame_dict_host writes
 *   zmt_zstd_decompress_dict_device     zmt_zstd_decompress_device against the dictionary
 * The calls without a dictionary keep refusing a frame that names a Dictionary_ID with ZMT_ST_UNSUPPORTED, and so does
 * the segment walk (zmt_zstd_segment_host). */
#define ZF_DICT 8u                   /* d_frame_seq: the frame decodes against the batch's dictionary */
typedef struct {
    uint32_t status;             /* ZMT_ST_OK, ZMT_ST_BAD_HEADER (unusable tables / repeat offsets), ZMT_ST_TRUNCATED */
    uint32_t dict_id;            /* 0 for raw content */
    uint32_t kind;               /* 0 raw content, 1 formatted */
    uint32_t reserved;
    uint64_t content_bytes;      /* history the frames may reach */
    uint64_t content_off;        /* where the content starts in the dictionary */
} zmt_zstd_dict_info;
size_t zmt_zstd_ddict_bytes(void);
int    zmt_zstd_ddict_load_device(const void* d_dict, uint64_t dict_bytes, void* d_ddict, zmt_zstd_dict_info* d_info, void* stream);
int    zmt_zstd_scan_frame_dict_host(const uint8_t* frame, size_t n, uint64_t base_off, uint32_t frame_idx, void* blocks_out,
                                     uint32_t* nblocks_io, uint32_t max_blocks, uint64_t* scratch_used, uint64_t* content_size,
                                     uint32_t* needs_seq, const zmt_zstd_dict_info* dict);
int    zmt_zstd_index_dict_device(const void* d_in, uint64_t in_bytes, uint32_t max_frames, uint64_t* d_frame_off, uint32_t* d_frame_csize,
                                  uint32_t* d_frame_first_blk, uint64_t* d_frame_scratch, uint64_t* d_expect, uint32_t* d_frame_seq,
                                  uint64_t* d_out_off, zmt_frame_index* d_info, void* d_work, void* stream, const void* d_ddict);
int    zmt_zstd_index_plain_dict_device(const void* d_in, uint64_t in_bytes, uint32_t max_frames, uint64_t* d_frame_off, uint32_t* d_frame_csize,
                                        uint32_t* d_frame_first_blk, uint64_t* d_frame_scratch, uint64_t* d_expect, uint32_t* d_frame_seq,
                                        uint64_t* d_out_off, zmt_frame_index* d_info, void* d_work, void* stream, const void* d_ddict);
int    zmt_zstd_blocks_dict_device(const void* d_in, uint32_t nframes, const uint64_t* d_frame_off, const uint32_t* d_frame_csize,
                                   const uint32_t* d_frame_first_blk, const uint64_t* d_frame_scratch, void* d_blocks, uint32_t nblocks, void* stream,
                                   const void* d_ddict);
int    zmt_zstd_decompress_dict_device(const void* d_in, const void* d_blocks, uint32_t nblocks, const uint32_t* d_frame_first_blk,
                                       const uint64_t* d_expect, const uint32_t* d_frame_seq, uint32_t nframes, void* d_out,
                                       const uint64_t* d_out_off, uint64_t* d_out_size, uint32_t* d_status, void* d_work, void* stream,
                                       const void* d_ddict);

/* ---- Compressing against a zstd dictionary (levels 6-22) ----
 * zmt_zstd_cdict_build_device indexes the content of a dictionary that zmt_zstd_ddict_load_device has loaded into
 * d_ddict, on the same stream: it reads the content's address and size from the record on the device (no round trip),
 * hashes every position q with q + 5 <= the content's length as the search class hashes a chunk's, sorts them, and
 * writes the opaque index d_cdict (zmt_zstd_cdict_bytes(dict_bytes) bytes of device memory: a 16 MiB head table,
 * 4 bytes per dictionary byte for the chains and 16 more plus the sort's scratch while it builds).  dict_bytes is the
 * size the dictionary was loaded with; 2^31 or more is ZMT_ST_BAD_ARG (zmt_zstd_cdict_bytes returns 0).  An index built
 * on a record whose load failed is empty and names no Dictionary_ID: the frames are those of the call without a
 * dictionary (the load's zmt_zstd_dict_info reports the failure).  The index keeps the addresses of the record and of
 * the dictionary's bytes; both must outlive every call that names it.  Reports under ZMT_K_ZL_HASH / ZMT_K_ZL_SORT.
 *
 * zmt_zstd_compress_dict_device is zmt_zstd_compress_level_device with the index: same layout contract, workspace
 * (zmt_zstdc_level_workspace_bytes at the same level) and output bound.  A chunk's hash chain that runs out with steps
 * and window left continues through the dictionary's content, which sits before every chunk (zstd_lazy_rule.h): matches
 * may start up to the window behind the chunk's start and end at the content's end at the latest.  Every offset is
 * written explicitly and the sequence tables are the predefined ones, so a frame uses only the dictionary's content; a
 * formatted dictionary's ID (not 0) is named in the frame header in 1, 2 or 4 bytes as libzstd writes it, which
 * zmt_zstdc_out_bound's per-window slack covers.  Levels 1-5 are ZMT_ST_BAD_ARG (the level-3 class has no chains);
 * d_cdict = NULL is the call without a dictionary, byte for byte. */
size_t zmt_zstd_cdict_bytes(uint64_t dict_bytes);
int    zmt_zstd_cdict_build_device(const void* d_ddict, uint64_t dict_bytes, void* d_cdict, void* stream);
int    zmt_zstd_compress_dict_device(const void* d_in, uint64_t in_bytes, uint32_t chunk_size, const uint32_t* d_chunk_bytes,
                                     uint32_t nchunks, int level, void* d_work, void* d_out, uint64_t* d_frame_off,
                                     void* stream, const void* d_cdict);

/* ---- LZ4F frames of any size in bounded memory ----
 * An LZ4F frame of any size, decoded as a chain of segments, each a run of whole blocks (what LZ4F_decompress does
 * through two fixed buffers when the reference streams a plain .lz4 file, lib/lz4-mt_decompress.c:391-483).  Frame f of
 * a zmt_lz4_decompress_segments_device batch is then a segment whose bytes start at d_in + d_frame_off[f] + 12:
 *   - the first segment starts with the frame header, a later one with a block header (no LZ4F header);
 *   - the last segment ends with the end mark and the content checksum, an earlier one right behind a block;
 *   - its content goes to d_out + d_out_off[f]; in a linked-block frame the last `history` bytes the frame decoded so
 *     far (up to 64 KiB) must lie directly below, in place before the call.
 * Between segments, d_seg[f] carries the frame's state on the device.  The caller zeroes it before the first segment
 * and sets `flags` and `history` for every segment; the device owns the other fields: the first segment records FLG,
 * BD and the content size from the header, every segment folds its bytes into the running XXH32 and advances
 * `produced`.  The content checksum and the content size are checked on the last segment only.  d_out_size[f] is the
 * segment's decoded size.  zmt_lz4f_segment_host finds a segment's end.  A frame with FIRST | LAST is a whole frame. */
#define ZMT_SEG_FIRST 1u
#define ZMT_SEG_LAST  2u
typedef struct {
    uint64_t history;         /* in: decoded bytes of the frame directly below d_out + d_out_off[f] (0 for the first segment) */
    uint64_t produced;        /* device: content bytes of the frame's segments so far */
    uint64_t content_size;    /* device: the header's content size, ~0 without one */
    uint32_t flags;           /* in: ZMT_SEG_* */
    uint8_t  flg, bd;         /* device: the frame's FLG / BD bytes */
    uint16_t pending_len;     /* device: bytes in pending[] */
    uint32_t acc[4];          /* device: XXH32 accumulators */
    uint8_t  pending[16];     /* device: content bytes not yet folded into acc[] */
} zmt_lz4_segment;
int      zmt_lz4_decompress_segments_device(const void* d_in, uint64_t in_bytes, const uint64_t* d_frame_off, const uint32_t* d_frame_csize,
                                            uint32_t nframes, uint32_t nslots, void* d_out, const uint64_t* d_out_off, uint64_t* d_out_size,
                                            uint32_t* d_status, zmt_lz4_segment* d_seg, void* d_work, void* stream);
/* Host walk of one segment: seg[0..n) holds the segment's bytes as far as they are known, its first block header at
 * seg[start] (start = the header length for the first segment, else 0); flg / bd are the frame's FLG / BD bytes.  The
 * segment runs to the first block boundary at or past seg + max_in, or to where its blocks reach max_out bytes of room,
 * or to the frame's end, and holds at least one block or the end mark.  *end = its length, *room = the output room it
 * needs (blockMaxSize per compressed block), *last = 1 if it ends the frame.  Returns ZMT_ST_OK, or ZMT_ST_TRUNCATED when
 * the segment's bytes are not all in seg[0..n) yet (read on). */
int      zmt_lz4f_segment_host(const uint8_t* seg, size_t n, size_t start, uint32_t flg, uint32_t bd, size_t max_in, uint64_t max_out,
                               size_t* end, uint64_t* room, uint32_t* last);

/* ---- zstd frames of any size in bounded memory ----
 * A zstd frame decoded as a chain of segments, each a run of whole blocks (what ZSTD_decompressStream does through two
 * fixed buffers when the reference streams a plain .zst file, lib/zstd-mt_decompress.c:552-687).  Four kinds of state
 * cross a cut:
 *   - the window: matches of a segment may reach up to Window_Size bytes back, into earlier segments;
 *   - the repeat offsets;
 *   - the tables a block may inherit (treeless literals, Repeat_Mode sequence tables): the block that last described the
 *     Huffman tree and the last FSE / RLE describer of each of the LL, OF and ML tables — at most four blocks;
 *   - the XXH64 content checksum and the content size.
 *
 * zmt_zstd_segment_host walks one segment on the host, resuming where the walk state `w` stands (zero it for a new
 * frame).  seg[0..n) holds the frame's bytes from frame offset w->pos on, as far as they are known; base_off is where
 * seg[0] lies in the decoder's input.  The segment runs to the first block boundary at or past seg + max_in, or to where
 * its blocks reach max_out bytes of room, or to the frame's end, and holds at least one block.  Its descriptors go to
 * blocks_out[*nblocks_io...] (below max_blocks), scratch from *scratch_used on, as for zmt_zstd_scan_frame_host.  A later
 * segment first gets one descriptor per table source it carries (zmt_zstd_segment_sources): type 3, no content, never
 * decoded or executed, named by the blocks that inherit its tables.  Their bytes must lie directly below seg[0] in the
 * decoder's input, in the order the sources are listed.  On ZMT_ST_OK: *end = the segment's length, *room = the output
 * room it needs (128 KiB per compressed block), *flags = the ZF bits for d_frame_seq (the dependent-block route is always
 * set), *last = 1 if it ends the frame (content checksum included), and `w` stands at the next segment.  ZMT_ST_TRUNCATED:
 * the segment's bytes are not all in seg[0..n) yet (read on); `w` is unchanged then, as on any other error. */
typedef struct {
    uint64_t pos;             /* frame offset of the next block header (0: the frame header comes first) */
    uint64_t content_size;    /* Frame_Content_Size, ~0 without one */
    uint64_t window;          /* Window_Size (RFC 8878 3.1.1.1.2; Frame_Content_Size for a Single_Segment frame) */
    uint32_t flags;           /* ZF bits of the frame so far: 1 dependent blocks, 2 content checksum, 4 no content size */
    uint32_t nblk;            /* blocks of the frame walked so far */
    uint32_t done;            /* 1: the frame's last block and checksum were walked */
    uint32_t reserved;
    /* the four table sources: 0 the Huffman tree, 1-3 the LL / OF / ML tables.  src_off = frame offset of the describing
     * block's content, src_len = its size; src_off = ~0: none yet, ~1: the predefined table (sequence tables only) */
    uint64_t src_off[4];
    uint32_t src_len[4];
} zmt_zstd_walk;
int      zmt_zstd_segment_host(const uint8_t* seg, size_t n, uint64_t base_off, uint32_t frame_idx, zmt_zstd_walk* w,
                               size_t max_in, uint64_t max_out, void* blocks_out, uint32_t* nblocks_io, uint32_t max_blocks,
                               uint64_t* scratch_used, size_t* end, uint64_t* room, uint32_t* flags, uint32_t* last);
/* The table sources a segment starting at `w` carries: distinct describing blocks in frame order, off[i] / len[i] (frame
 * offset and size of block i's content, at most four).  Returns their count; their bytes, back to back, are the carry
 * area below the segment. */
uint32_t zmt_zstd_segment_sources(const zmt_zstd_walk* w, uint64_t* off, uint32_t* len);
/* Decoding: the arguments of zmt_zstd_decompress_device, every frame of the batch a segment.  d_seg[f] carries frame f's
 * state: the caller zeroes it before the first segment and sets `flags` and `history` for every segment; the device
 * owns the other fields.  Segment f's content goes to d_out + d_out_off[f]; the last `history` bytes the frame decoded so
 * far (min(Window_Size, produced)) must lie directly below, in place before the call.  d_expect[f] of a first segment is
 * the frame's content size (~0 without one), kept in the record; a later segment's entry is not read.  d_frame_seq[f]
 * must carry the dependent-block bit (zmt_zstd_segment_host sets it).  Every segment seeds the repeat offsets from the
 * record and stores them back, and folds its content into the running XXH64; the content size and the content checksum
 * are checked on the last segment.  d_out_size[f] is the segment's decoded size.  A segment with FIRST | LAST is a whole
 * frame. */
typedef struct {
    uint64_t history;         /* in: decoded bytes of the frame directly below d_out + d_out_off[f] (0 for the first segment) */
    uint64_t produced;        /* device: content bytes of the frame's segments so far */
    uint64_t content_size;    /* device: the header's content size, ~0 without one */
    uint32_t flags;           /* in: ZMT_SEG_* */
    uint32_t rep[3];          /* device: the repeat offsets behind the segments so far */
    uint64_t acc[4];          /* device: XXH64 accumulators */
    uint32_t pending_len;     /* device: bytes in pending[] */
    uint32_t reserved;
    uint8_t  pending[32];     /* device: content bytes not yet folded into acc[] */
} zmt_zstd_segment;
int      zmt_zstd_decompress_segments_device(const void* d_in, const void* d_blocks, uint32_t nblocks, const uint32_t* d_frame_first_blk,
                                             const uint64_t* d_expect, const uint32_t* d_frame_seq, uint32_t nframes, void* d_out,
                                             const uint64_t* d_out_off, uint64_t* d_out_size, uint32_t* d_status, zmt_zstd_segment* d_seg,
                                             void* d_work, void* stream);

/* ---- Range reads: byte ranges of a stream's content, decoding only the frames that hold them ----
 * On top of the device index above (container or plain; for a plain stream pass d_in - 12 as to the decode calls).  The
 * unit of access is the frame: a frame's content is only known by decoding it whole, so every frame a range touches is
 * decoded once per batch, however many ranges touch it, and every other frame is not read at all.
 *
 * Content table, once per stream: d_content_off[0..nframes] = the exclusive prefix of the frames' content sizes, each
 * from the frame's own header (LZ4F FLG bit 3 + LE64 field; zstd Frame_Content_Size, i.e. d_expect of the zstd index).
 * The summary is a zmt_frame_index: status, bad_frame (nframes when OK), bad_offset = d_frame_off[bad_frame],
 * nframes, out_bytes = the total content; nblocks and scratch_bytes are 0.  status:
 *   ZMT_ST_UNSUPPORTED   a frame without a content size (the lz4 CLI's default, zstd written to a pipe): its content
 *                        position cannot be known without decoding every frame before it
 *   ZMT_ST_CONTENT_SIZE  a stated content size above 32768 bytes per compressed byte, more than either format can
 *                        produce: a damaged header, which would wrap the table
 * The first such frame in stream order is named.  d_work: zmt_range_workspace_bytes(nframes, 0).
 *
 * Plan, once per batch: d_ranges = nranges pairs {start, length} in content coordinates, in any order, overlapping,
 * repeated or empty.  A range [start, start + length) is bad (ZMT_ST_BAD_ARG) when it ends past the content or
 * start + length overflows; a bad range takes no room in dst.  The plan finds the frames each good range touches, marks
 * them, and writes the decode tables of the marked frames (the "selected" frames, in stream order) into d_work, which
 * must then stay untouched until the batch's read call.  d_dst_off[0..nranges] = the exclusive prefix of the lengths of
 * the good ranges: range r's bytes go to dst + d_dst_off[r].  The host reads back the zmt_range_plan summary and sizes
 * the read's buffers from it; the workspace only depends on nframes and nranges.
 *
 * Read, once per batch, with the plan's d_work and a host copy of its summary:
 *   LZ4    a kernel packs the selected frames (a 12-byte container header and the payload each) into the read
 *          workspace, and zmt_lz4_decompress_device decodes that packed stream, so its match records cover only the
 *          selected frames' compressed bytes, not the stream's;
 *   zstd   zmt_zstd_blocks_device builds the selected frames' block table and zmt_zstd_decompress_device decodes them
 *          in place in d_in (its workspace does not depend on the input's size);
 * both decode into d_scratch (plan.scratch_bytes: the selected frames' content back to back), then a gather kernel
 * copies every good range to dst + d_dst_off[r] (any alignment) in pieces of at most 64 KiB.  d_range_status[r]:
 *   ZMT_ST_OK, ZMT_ST_BAD_ARG for a bad range (its dst bytes are not written), or the decoder's status of the first frame
 *   the range touches that failed (BLOCK, CONTENT_CHECKSUM, ...; its dst bytes are not written).
 * Selected frames are decoded whole, so their content checksums (and LZ4F block checksums) are verified as in a
 * whole-stream decode.  A damaged frame no range of the batch touches is not decoded, and so its damage is not reported.
 * Memory per batch: the plan's workspace is O(nframes + nranges); the read's workspace (zmt_*_range_read_workspace_bytes)
 * and d_scratch are O(selected compressed bytes + selected content), never O(stream):
 *   LZ4    256-aligned packed_bytes + zmt_lz4d_workspace_bytes(nsel, nunits, packed_bytes)
 *   zstd   256-aligned nunits * zmt_zstd_blk_desc_bytes() + zmt_zstdd_workspace_bytes(nsel, nunits, dec_scratch)
 * All calls return ZMT_ST_OK once enqueued, ZMT_ST_BAD_ARG or ZMT_ST_CUDA. */
typedef struct {
    uint32_t status;        /* ZMT_ST_OK, or ZMT_ST_BAD_ARG when a range is bad (the other ranges are planned and read) */
    uint32_t bad_range;     /* the first bad range (== nranges when none) */
    uint32_t nframes;       /* the plan's arguments, for the read call */
    uint32_t nranges;
    uint32_t nsel;          /* selected frames: the frames the good ranges touch */
    uint32_t nunits;        /* LZ4: block-table slots of the selected frames; zstd: their blocks */
    uint64_t packed_bytes;  /* LZ4: bytes of the packed stream of the selected frames (0 for zstd) */
    uint64_t scratch_bytes; /* the selected frames' content: the size of d_scratch */
    uint64_t dec_scratch;   /* zstd: the selected frames' entropy scratch (third argument of zmt_zstdd_workspace_bytes) */
    uint64_t dst_bytes;     /* d_dst_off[nranges]: the size of dst */
    uint64_t npieces;       /* gather pieces (at most 64 KiB each) */
} zmt_range_plan;

size_t   zmt_range_workspace_bytes(uint32_t nframes, uint32_t nranges);
int      zmt_lz4_content_offsets_device(const void* d_in, uint32_t nframes, const uint64_t* d_frame_off, const uint32_t* d_frame_csize,
                                        uint64_t* d_content_off, zmt_frame_index* d_info, void* d_work, void* stream);
int      zmt_zstd_content_offsets_device(uint32_t nframes, const uint64_t* d_frame_off, const uint32_t* d_frame_csize, const uint64_t* d_expect,
                                         uint64_t* d_content_off, zmt_frame_index* d_info, void* d_work, void* stream);
int      zmt_lz4_range_plan_device(uint32_t nframes, const uint32_t* d_frame_csize, const uint64_t* d_content_off, const uint64_t* d_ranges,
                                   uint32_t nranges, uint64_t* d_dst_off, zmt_range_plan* d_plan, void* d_work, void* stream);
int      zmt_zstd_range_plan_device(uint32_t nframes, const uint32_t* d_frame_csize, const uint32_t* d_frame_first_blk, const uint64_t* d_frame_scratch,
                                    const uint64_t* d_content_off, const uint64_t* d_ranges, uint32_t nranges, uint64_t* d_dst_off,
                                    zmt_range_plan* d_plan, void* d_work, void* stream);
size_t   zmt_lz4_range_read_workspace_bytes(const zmt_range_plan* plan);
size_t   zmt_zstd_range_read_workspace_bytes(const zmt_range_plan* plan);
int      zmt_lz4_range_read_device(const void* d_in, const uint64_t* d_frame_off, const uint32_t* d_frame_csize, const zmt_range_plan* plan,
                                   void* d_dst, const uint64_t* d_dst_off, uint32_t* d_range_status, void* d_scratch, void* d_read_work,
                                   void* d_work, void* stream);
int      zmt_zstd_range_read_device(const void* d_in, const uint64_t* d_frame_off, const uint32_t* d_frame_csize, const uint64_t* d_expect,
                                    const uint32_t* d_frame_seq, const zmt_range_plan* plan, void* d_dst, const uint64_t* d_dst_off,
                                    uint32_t* d_range_status, void* d_scratch, void* d_read_work, void* d_work, void* stream);

/* ---- multi-GPU: one LZ4MT_* / ZSTDCB_* call deals its batches round-robin over the devices named by the
 * environment variable ZSTDMT_GPUS ("all" or "0,1,..."; default: the calling thread's current device) and re-serialises
 * the frames on the host.  zmt_device_batches(dev) = batches submitted to that device since the library was loaded. */
uint64_t zmt_device_batches(int dev);

/* ---- per-kernel device timing (CUDA events on the launching stream) ----
 * zmt_prof_begin() arms it; every kernel launched by the entry points above is bracketed by two
 * events; zmt_prof_end() (after the caller synchronised the stream) sums them per kernel id. */
enum { ZMT_K_LZ4_COMPRESS = 0, ZMT_K_XXH32, ZMT_K_LZ4_SIZES, ZMT_K_SCAN, ZMT_K_LZ4_PACK, ZMT_K_LZ4_DECODE, ZMT_K_XXH32_DEC,
       ZMT_K_ZSTD_COMPRESS, ZMT_K_ZSTD_PACK, ZMT_K_ZSTD_DECODE, ZMT_K_LZ4_DEXEC,
       ZMT_K_ZL_HASH, ZMT_K_ZL_SORT, ZMT_K_ZL_SEARCH, ZMT_K_ZL_BLOCKS, ZMT_K_L4H_BLOCKS, ZMT_K_FRAME_INDEX, ZMT_K_COUNT };
/* LZ4 decode: ZMT_K_LZ4_DECODE = pass A (token parse + literals), ZMT_K_LZ4_DEXEC = pass B (match execution)
 * zstd levels 6-22: ZMT_K_ZL_HASH = hash, ZMT_K_ZL_SORT = radix sort + prev[], ZMT_K_ZL_SEARCH = chain walk,
 * ZMT_K_ZL_BLOCKS = lazy parse + entropy stage (the frame pack stays ZMT_K_ZSTD_PACK)
 * LZ4 levels 10-12: hash, sort and search as zstd's (ZMT_K_ZL_HASH / SORT / SEARCH), ZMT_K_L4H_BLOCKS = lazy parse +
 * LZ4 sequences; checksum, sizes, scan and pack as level 1's
 * ZMT_K_FRAME_INDEX = one index call (container or plain walk, frame pass, scans, summary) or one zmt_zstd_blocks_device call;
 * range reads report here too, as the index's consumers: one content-table or plan call, and the pack stage and the
 * status + gather stage of a read call (the decoders inside a read call report under their own ids) */
void zmt_prof_begin(void);
int  zmt_prof_end(double* ms, int* count, int max_ids);

#ifdef __cplusplus
}
#endif
#endif
