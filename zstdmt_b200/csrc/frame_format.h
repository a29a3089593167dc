// frame_format.h — the header formats the decoders read, in one place for the host and the device.
//
// The host pipeline (host_api.cpp, zmt_zstd_scan_frame_host in zstd_decode.cu) and the device frame index
// (frame_index.cu) both call these walkers, so the block table the zstd decoder takes and the room the LZ4 decoder
// gets per frame are defined once.  Every read stays inside [p, p + n): the fields come from outside the program.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include "zmt_dev.h"

#ifdef __CUDACC__
#define ZMT_HD __host__ __device__ __forceinline__
#else
#define ZMT_HD inline
#endif

#define ZMT_CONTAINER_MAGIC 0x184D2A50u      // [LE32 magic][LE32 4][LE32 payload size] before every frame
#define ZMT_LZ4F_MAGIC      0x184D2204u
#define ZMT_ZSTD_MAGIC      0xFD2FB528u

ZMT_HD uint32_t zf_rd32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
ZMT_HD uint64_t zf_rd64(const uint8_t* p) { return (uint64_t)zf_rd32(p) | ((uint64_t)zf_rd32(p + 4) << 32); }
ZMT_HD uint32_t zf_rd24(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16); }

// ---------------------------------------------------------------- LZ4F
// Bytes of an LZ4F frame header with this FLG byte: magic, FLG, BD, [content size], [dictionary ID], header checksum.
ZMT_HD size_t lz4f_header_len(uint32_t flg) { return 4 + 2 + ((flg & 8) ? 8 : 0) + ((flg & 1) ? 4 : 0) + 1; }

// A block walk that can stop at a block boundary and resume there (a frame decoded as a chain of segments).
struct Lz4fWalk {
    size_t   pos;               // offset in the frame of the next block header (start: lz4f_header_len)
    uint64_t bound;             // the most the blocks walked so far decode to (blockMaxSize per compressed block)
    uint32_t nblk;              // blocks walked so far
    uint32_t done;              // 1: the end mark was met; pos = the frame's length, content checksum included
};

// Walks block headers of the LZ4F frame p[0..n) with FLG / BD from w->pos on, and stops at the first block boundary at
// or past pos_stop or where the bound reaches bound_stop, or at the frame's end (w->done).  Returns false if a block
// header lies past n ("need more bytes"); w then stands behind the last header read, whose block may itself run past n.
// Only headers are read: a caller that cuts the frame at w->pos checks that w->pos <= n.
ZMT_HD bool lz4f_walk_blocks(const uint8_t* p, size_t n, uint32_t flg, uint32_t bd, Lz4fWalk* w, size_t pos_stop, uint64_t bound_stop)
{
    const uint64_t blkmax = 1ull << (8 + 2 * ((bd >> 4) & 7));
    for (;;) {
        if (w->pos >= pos_stop || w->bound >= bound_stop) return true;
        if (w->pos + 4 > n) return false;
        const uint32_t bh = zf_rd32(p + w->pos); w->pos += 4;
        if (bh == 0) { w->pos += (flg & 4) ? 4 : 0; w->done = 1; return true; }
        const uint32_t bs = bh & 0x7FFFFFFFu;
        w->bound += (bh & 0x80000000u) ? bs : blkmax;
        w->pos += (size_t)bs + ((flg & 0x10) ? 4 : 0);
        w->nblk++;
    }
}

// Walks an LZ4F frame's header and block headers in p[0..n) (n >= 7): *len = the frame's length, content checksum
// included; *bound = the most its blocks decode to (blockMaxSize per compressed block).  false: the block headers run
// past n (*bound then covers the blocks before the cut).
ZMT_HD bool lz4f_walk(const uint8_t* p, size_t n, size_t* len, uint64_t* bound)
{
    Lz4fWalk w; w.pos = lz4f_header_len(p[4]); w.bound = 0; w.nblk = 0; w.done = 0;
    const bool ok = lz4f_walk_blocks(p, n, p[4], p[5], &w, ~(size_t)0, ~0ull);
    *bound = w.bound;
    if (ok) *len = w.pos;
    return ok;
}

// The content size an LZ4F frame's header states: p[0..n) = the frame from its magic.  true: FLG bit 3 is set and the
// 8-byte field lies inside p[0..n), *cs = its value (untrusted).  false: not an LZ4F frame, no such field, or the header
// is cut short before it.  Both the decoders' room rule below and the range reads' content table read it here.
ZMT_HD bool lz4f_content_size(const uint8_t* p, size_t n, uint64_t* cs)
{
    if (n < 15 || zf_rd32(p) != ZMT_LZ4F_MAGIC || !(p[4] & 0x08)) return false;
    *cs = zf_rd64(p + 6);
    return true;
}

// The content size of an LZ4F frame known without decoding it: the header's field, or 0 for a frame without one whose
// first block header is the end mark (liblz4 states no content size for an empty input).  false: neither.
ZMT_HD bool lz4f_known_content_size(const uint8_t* p, size_t n, uint64_t* cs)
{
    if (lz4f_content_size(p, n, cs)) return true;
    if (n < 7 || zf_rd32(p) != ZMT_LZ4F_MAGIC) return false;
    const size_t h = lz4f_header_len(p[4]);
    if (n < h + 4 || zf_rd32(p + h) != 0) return false;
    *cs = 0;
    return true;
}

// The room one LZ4 payload of n bytes gets in the output, from its own header (pt_decompress sizes the buffer from
// LE64 @ payload+6, lz4-mt_decompress.c:329-335).  Returns false if the header is unusable (ZMT_ST_BAD_HEADER).
// A payload without the LZ4F magic gets room 0: the decoder reports its precise status.
ZMT_HD bool lz4f_out_size(const uint8_t* p, size_t n, uint64_t* out)
{
    if (n < 7 || zf_rd32(p) != ZMT_LZ4F_MAGIC) { *out = 0; return true; }
    const uint32_t flg = p[4], bd = p[5];
    if (flg & 0x08) {
        uint64_t v = 0;
        if (!lz4f_content_size(p, n, &v)) return false;
        // untrusted field: LZ4 cannot expand by more than 255x, anything larger is a corrupt header (the reference
        // fails its malloc there); without this bound a huge value would wrap the running output offsets
        if (v > (uint64_t)n * 255 + 65536) return false;
        *out = v; return true;
    }
    // no content-size field: bound it by walking the block headers (each block <= blockMaxSize)
    if (((bd >> 4) & 7) < 4) return false;
    size_t len = 0;
    lz4f_walk(p, n, &len, out);
    return true;
}

// LZ4 decoder block-table slots a frame with this much room takes (the nslots argument sums them)
ZMT_HD uint64_t lz4_frame_slots(uint64_t room) { const uint64_t nb = (room + 65535) / 65536; return nb ? nb : 1; }

// ---------------------------------------------------------------- plain streams
// An ordinary .lz4 / .zst file: codec frames and skippable frames (magic 0x184D2A50..0x184D2A5F, LE32 size, payload) back
// to back, without container headers.  A frame's end is only known by walking its block headers.  The host's plain path
// (decompress_single_stream) and the device's plain index (frame_index.cu) take the same decision at every frame start
// from the two functions below and, for a zstd frame, zstd_frame_walk.

// The first decision at a frame start: p[0..n) = the stream's bytes from there.  ZMT_ST_OK: *skip = the length of a
// skippable frame (8 + its size), or 0 for a codec frame whose head is usable.  ZMT_ST_TRUNCATED: fewer than 4 bytes, a
// skippable frame whose size runs past n, or an LZ4F header shorter than 7 bytes.  ZMT_ST_BAD_MAGIC: neither a skippable
// frame nor the codec's magic (zstd: 0xFD2FB522..0xFD2FB528; the walk then rejects the legacy versions with BAD_MAGIC).
// ZMT_ST_BAD_HEADER: an LZ4F FLG version other than 01, or a block-size id below 4.
ZMT_HD int plain_frame_head(const uint8_t* p, size_t n, bool zstd, uint64_t* skip)
{
    *skip = 0;
    if (n < 4) return ZMT_ST_TRUNCATED;
    const uint32_t magic = zf_rd32(p);
    if ((magic & 0xFFFFFFF0u) == ZMT_CONTAINER_MAGIC) {
        if (n < 8 || n - 8 < zf_rd32(p + 4)) return ZMT_ST_TRUNCATED;
        *skip = 8 + (uint64_t)zf_rd32(p + 4);
        return ZMT_ST_OK;
    }
    if (zstd) return magic >= 0xFD2FB522u && magic <= ZMT_ZSTD_MAGIC ? ZMT_ST_OK : ZMT_ST_BAD_MAGIC;
    if (magic != ZMT_LZ4F_MAGIC) return ZMT_ST_BAD_MAGIC;
    if (n < 7) return ZMT_ST_TRUNCATED;
    if ((p[4] >> 6) != 1 || ((p[5] >> 4) & 7) < 4) return ZMT_ST_BAD_HEADER;
    return ZMT_ST_OK;
}

// The rest of the decision for an LZ4F frame whose head passed: p[0..n) = the stream's bytes from the frame start.
// ZMT_ST_OK: *len = the frame's length (content checksum included), *room = its content size, or the block bound
// (blockMaxSize per compressed block) without one.  ZMT_ST_TRUNCATED: the header or a block runs past n; *stop = the
// block header the walk could not read, or n.  ZMT_ST_CONTENT_SIZE: a content size above the block bound (*stop = 0):
// the field is untrusted, and a plain frame has no payload size to bound it by but its own blocks.
ZMT_HD int lz4f_plain_frame(const uint8_t* p, size_t n, uint64_t* len, uint64_t* room, uint64_t* stop)
{
    Lz4fWalk w; w.pos = lz4f_header_len(p[4]); w.bound = 0; w.nblk = 0; w.done = 0;
    *stop = 0;
    if (!lz4f_walk_blocks(p, n, p[4], p[5], &w, ~(size_t)0, ~0ull) || w.pos > n) { *stop = w.pos < n ? w.pos : n; return ZMT_ST_TRUNCATED; }
    *len = w.pos; *room = w.bound;
    uint64_t cs = 0;
    if (lz4f_content_size(p, n, &cs)) {
        if (cs > w.bound) return ZMT_ST_CONTENT_SIZE;
        *room = cs;
    }
    return ZMT_ST_OK;
}

// ---------------------------------------------------------------- zstd block descriptors (the zstd decoder's block table)
#define ZB_RAW 0u
#define ZB_RLE 1u
#define ZB_CMP 2u
struct ZBlk {
    uint64_t comp_off;      // offset of the block CONTENT (after its 3-byte header) in the input buffer
    uint32_t comp_size;     // content bytes (1 for RLE)
    uint32_t frame;         // frame index in the batch
    uint32_t type;          // ZB_*
    uint32_t regen_hint;    // raw / RLE: regenerated size; compressed: literal bytes (regenerated)
    uint32_t nseq;          // compressed: number of sequences
    uint32_t first;         // 1 if first block of its frame
    uint64_t seq_off;       // scratch offsets (bytes) for this block's sequence records / literals
    uint64_t lit_off;
    // blocks whose tables come from an earlier block of the frame (treeless literals, Repeat_Mode sequence tables): index of
    // the block whose section header DESCRIBES the table in use (ZB_SELF / ZB_PREDEF / ZB_NONE otherwise) — found by the
    // frame walk, so that every block can be entropy-decoded on its own
    uint32_t huf_src, ll_src, of_src, ml_src;
};
#define ZB_SELF   0xFFFFFFFFu
#define ZB_PREDEF 0xFFFFFFFEu
#define ZB_NONE   0xFFFFFFFDu
#define ZB_DICT   0xFFFFFFFCu       // the table comes from the batch's dictionary (a formatted one: ZDDict's descriptions)
struct ZDSeq { uint32_t ll; uint32_t off; uint32_t ml; uint32_t pad; };

// per-frame flags (the d_frame_seq[] argument of zmt_zstd_decompress_device; ZF_DICT = 8 is in the public header)
#define ZF_NEEDS_SEQ 1u     // blocks depend on earlier blocks: frame-sequential entropy pass
#define ZF_CHECKSUM  2u     // 4-byte content checksum (low 32 bits of XXH64) follows the last block
#define ZF_NO_SIZE   4u     // no Frame_Content_Size: the reported size is an upper bound (128 KiB per compressed block)

// A loaded dictionary (zmt_zstd_ddict_load_device writes it; callers hold it as opaque device memory).  The walk reads
// only `info` (status, ID, kind), so the host scan takes the zmt_zstd_dict_info summary in its place.
struct ZDDict {
    zmt_zstd_dict_info info;
    uint64_t dict;              // device address of the dictionary's bytes (the caller's buffer)
    uint32_t rep[3];            // repeat offsets the frames start from
    uint32_t huf_off, of_off, ml_off, ll_off;     // formatted: where the four table descriptions start in the dictionary
    uint32_t rep_off;           // formatted: where the repeat offsets start (the LL description's end)
};

// segments (zmt_zstd_segment_host): a table source carried from an earlier segment.  Only its bytes are used, by the
// blocks that name it in *_src: regen 0, nseq 0, never decoded or executed.
#define ZB_SRC 3u
#define ZW_NONE   (~0ull)       // zmt_zstd_walk::src_off: no describer yet
#define ZW_PREDEF (~1ull)       // zmt_zstd_walk::src_off: the predefined table

// The table sources a segment starting at w carries: the distinct describing blocks of w->src_off, in frame order.
ZMT_HD uint32_t zstd_walk_sources(const zmt_zstd_walk* w, uint64_t* off, uint32_t* len)
{
    uint32_t k = 0;
    if (w->pos == 0) return 0;
    for (uint32_t t = 0; t < 4; t++) {
        const uint64_t o = w->src_off[t];
        bool dup = o >= ZW_PREDEF;
        for (uint32_t i = 0; i < k; i++) dup = dup || off[i] == o;
        if (dup) continue;
        uint32_t i = k++;
        for (; i > 0 && off[i - 1] > o; i--) { off[i] = off[i - 1]; len[i] = len[i - 1]; }
        off[i] = o; len[i] = w->src_len[t];
    }
    return k;
}

// Walks the blocks of one zstd frame from where *w stands: p[0..n) are the frame's bytes from frame offset w->pos on
// (w->pos == 0: the frame header comes first and resets *w), `base_off` = where p[0] lies in the decoder's input buffer.
// Stops at the first block boundary at or past p + pos_stop or where the blocks of this call reach bound_stop bytes of
// room (after one block at least), or at the frame's end (w->done, content checksum included).  A call that resumes a
// frame first emits one ZB_SRC descriptor per table source (zstd_walk_sources), whose bytes the caller places directly
// below p[0], in that order.  W = true writes one descriptor per block at blocks_out[*nblocks_io++] (below index
// max_blocks); W = false only counts them.  Either way *nblocks_io advances by the descriptor count, *scratch_used by the
// entropy scratch the blocks take (their seq_off / lit_off), w->flags collects the ZF_* bits, *bound gets the room of
// the call's blocks (128 KiB per compressed block).  w->pos = the frame offset the walk stopped at: the next block header,
// the frame's length at its end, or on failure the header element it could not take.  Returns ZMT_ST_*.
// dict: the batch's dictionary (D = true).  Without one a frame that names a Dictionary_ID is ZMT_ST_UNSUPPORTED.  With
// one every frame decodes against it (ZF_DICT | ZF_NEEDS_SEQ) unless it names another ID (ZMT_ST_DICT_WRONG, w->pos = 0),
// and a formatted dictionary is the describer of all four tables until a block of the frame describes its own (ZB_DICT).
// Only a whole-frame walk (w->pos == 0) takes a dictionary.  D = false: the walk without one, which never reads dict.
template <bool W, bool D = false>
ZMT_HD int zstd_walk_blocks(const uint8_t* p, size_t n, uint64_t base_off, uint32_t frame_idx, ZBlk* blocks_out,
                            uint32_t* nblocks_io, uint32_t max_blocks, uint64_t* scratch_used, zmt_zstd_walk* w,
                            size_t pos_stop, uint64_t bound_stop, uint64_t* bound, const zmt_zstd_dict_info* dict = nullptr)
{
    const uint64_t at0 = w->pos;
    size_t pos = 0;
    uint64_t bnd = 0;
    uint32_t walked = 0;
    *bound = 0;
    if (at0 == 0) {
        w->flags = 0; w->nblk = 0; w->done = 0; w->reserved = 0; w->content_size = ZW_NONE; w->window = 0;
        for (uint32_t t = 0; t < 4; t++) { w->src_off[t] = ZW_NONE; w->src_len[t] = 0; }
        if (n < 6 || zf_rd32(p) != ZMT_ZSTD_MAGIC) return n < 6 ? ZMT_ST_TRUNCATED : ZMT_ST_BAD_MAGIC;
        const uint32_t fhd = p[4], fcs = fhd >> 6, single = (fhd >> 5) & 1, did = fhd & 3;
        if (fhd & 0x08) return ZMT_ST_BAD_HEADER;
        if (did && !D) return ZMT_ST_UNSUPPORTED;                         // dictionaries: only against a loaded one
        pos = 5 + (single ? 0 : 1);
        if (D && did) {
            const size_t dl = did == 3 ? 4 : did;
            if (n < pos + dl) return ZMT_ST_TRUNCATED;
            const uint32_t id = dl == 1 ? p[pos] : dl == 2 ? (uint32_t)(p[pos] | (p[pos + 1] << 8)) : zf_rd32(p + pos);
            if (id != 0 && id != dict->dict_id) return ZMT_ST_DICT_WRONG;  // ZSTD_decompress_usingDict: a frame without an ID takes the dictionary
            pos += dl;
        }
        if (D) {
            if (dict->status != ZMT_ST_OK) return (int)dict->status;      // a dictionary whose load failed decodes nothing
            w->flags |= ZF_DICT | ZF_NEEDS_SEQ;
        }
        const size_t fl = fcs == 0 ? (single ? 1 : 0) : fcs == 1 ? 2 : fcs == 2 ? 4 : 8;
        if (n < pos + fl) return ZMT_ST_TRUNCATED;
        uint64_t cs = 0;
        if (fl == 1) cs = p[pos]; else if (fl == 2) cs = (uint64_t)(p[pos] | (p[pos + 1] << 8)) + 256;
        else if (fl == 4) cs = zf_rd32(p + pos); else if (fl == 8) cs = zf_rd64(p + pos);
        if (single) w->window = cs;                                       // RFC 8878 3.1.1.1.2
        else { const uint32_t wd = p[5]; const uint64_t wb = 1ull << (10 + (wd >> 3)); w->window = wb + (wb >> 3) * (wd & 7); }
        pos += fl;
        if (fhd & 0x04) w->flags |= ZF_CHECKSUM;                         // XXH64 content checksum after the last block (verified on the device)
        if (fl == 0) w->flags |= ZF_NO_SIZE;                              // streamed frame: size from the blocks (bound: 128 KiB per compressed block)
        else w->content_size = cs;
    }
    // block that describes the Huffman tree / each sequence table in use, as a descriptor index of this call
    uint32_t cur[4];
    for (uint32_t t = 0; t < 4; t++) cur[t] = w->src_off[t] == ZW_PREDEF ? ZB_PREDEF : (D && dict->kind ? ZB_DICT : ZB_NONE);
    if (at0 != 0) {
        uint64_t so[4]; uint32_t sl[4];
        const uint32_t ns = zstd_walk_sources(w, so, sl);
        uint64_t at = base_off;
        for (uint32_t i = 0; i < ns; i++) at -= sl[i];
        for (uint32_t i = 0; i < ns; i++) {
            if (*nblocks_io >= max_blocks) return ZMT_ST_DST_SMALL;
            ZBlk B = ZBlk();
            B.frame = frame_idx; B.type = ZB_SRC; B.comp_off = at; B.comp_size = sl[i];
            B.seq_off = B.lit_off = *scratch_used;
            B.huf_src = B.ll_src = B.of_src = B.ml_src = ZB_SELF;
            for (uint32_t t = 0; t < 4; t++) if (w->src_off[t] == so[i]) cur[t] = *nblocks_io;
            if (W) blocks_out[*nblocks_io] = B;
            (*nblocks_io)++;
            at += sl[i];
        }
    }
    uint32_t bh_next = 0;                                             // the next block header, when loaded ahead (have_next)
    bool have_next = false;
    for (;;) {
        w->pos = at0 + pos;
        if (walked && (pos >= pos_stop || bnd >= bound_stop)) { *bound = bnd; return ZMT_ST_OK; }
        if (n - pos < 3) return ZMT_ST_TRUNCATED;
        const uint32_t bh = have_next ? bh_next : zf_rd24(p + pos); pos += 3;
        have_next = false;
        const uint32_t last = bh & 1, type = (bh >> 1) & 3, bs = bh >> 3;
        if (type == 3 || bs > 128 * 1024) return ZMT_ST_BLOCK;
        if (*nblocks_io >= max_blocks) return ZMT_ST_DST_SMALL;
        ZBlk B = ZBlk();                                              // no padding: every byte is zeroed
        B.frame = frame_idx; B.type = type; B.first = w->nblk == 0 ? 1 : 0; B.comp_off = base_off + pos;
        bnd += type == ZB_CMP ? 128 * 1024 : bs;
        if (type == ZB_RAW) { if (n - pos < bs) return ZMT_ST_TRUNCATED; B.comp_size = bs; B.regen_hint = bs; pos += bs; }
        else if (type == ZB_RLE) { if (n - pos < 1) return ZMT_ST_TRUNCATED; B.comp_size = 1; B.regen_hint = bs; pos += 1; }
        else {
            if (n - pos < bs || bs < 2) return ZMT_ST_TRUNCATED;
            // the walk is a chain of dependent loads: the next block header's goes out before this block's section
            // headers are parsed, so a compressed block costs one load latency, not three
            if (!last && n - pos - bs >= 3) { bh_next = zf_rd24(p + pos + bs); have_next = true; }
            const uint8_t* s = p + pos;
            const uint32_t b0 = s[0], lt = b0 & 3, sf = (b0 >> 2) & 3;
            uint32_t lregen, lcomp, lhdr;
            if (lt < 2) {
                if (sf == 0 || sf == 2) { lregen = b0 >> 3; lhdr = 1; }
                else if (sf == 1) { if (bs < 2) return ZMT_ST_BLOCK; lregen = (b0 >> 4) | ((uint32_t)s[1] << 4); lhdr = 2; }
                else { if (bs < 3) return ZMT_ST_BLOCK; lregen = (b0 >> 4) | ((uint32_t)s[1] << 4) | ((uint32_t)s[2] << 12); lhdr = 3; }
                lcomp = lt == 0 ? lregen : 1;
            } else {
                if (bs < 5) return ZMT_ST_BLOCK;
                if (sf < 2) { const uint32_t v = s[0] | (s[1] << 8) | ((uint32_t)s[2] << 16); lregen = (v >> 4) & 0x3FF; lcomp = (v >> 14) & 0x3FF; lhdr = 3; }
                else if (sf == 2) { const uint32_t v = zf_rd32(s); lregen = (v >> 4) & 0x3FFF; lcomp = (v >> 18) & 0x3FFF; lhdr = 4; }
                else { const uint64_t v = (uint64_t)zf_rd32(s) | ((uint64_t)s[4] << 32); lregen = (uint32_t)((v >> 4) & 0x3FFFF); lcomp = (uint32_t)((v >> 22) & 0x3FFFF); lhdr = 5; }
            }
            if ((uint64_t)lhdr + lcomp + 1 > bs) return ZMT_ST_BLOCK;
            const uint8_t* q = s + lhdr + lcomp; const uint32_t qn = bs - lhdr - lcomp;
            uint32_t nseq; const uint32_t q0 = q[0];
            if (q0 == 0) nseq = 0; else if (q0 < 128) nseq = q0;
            else if (q0 < 255) { if (qn < 2) return ZMT_ST_BLOCK; nseq = ((q0 - 128) << 8) + q[1]; }
            else { if (qn < 3) return ZMT_ST_BLOCK; nseq = q[1] + (q[2] << 8) + 0x7F00; }
            // state across blocks visible in the headers: treeless literals, FSE-coded weights are fine block-parallel,
            // any non-predefined sequence table mode may be followed by Repeat_Mode -> frame-sequential pass
            {
                const uint32_t used = q0 == 0 ? 1u : q0 < 128 ? 1u : q0 < 255 ? 2u : 3u;
                if (lt == 3) w->flags |= ZF_NEEDS_SEQ;
                if (nseq && qn > used && q[used] != 0) w->flags |= ZF_NEEDS_SEQ;
                const uint32_t me = *nblocks_io;
                B.huf_src = ZB_SELF;
                if (lt == 2) { cur[0] = me; w->src_off[0] = at0 + pos; w->src_len[0] = bs; }
                else if (lt == 3) B.huf_src = cur[0];
                B.ll_src = B.of_src = B.ml_src = ZB_SELF;
                if (nseq && qn > used) {
                    uint32_t src[3];
#pragma unroll
                    for (uint32_t t = 0; t < 3; t++) {
                        const uint32_t mode = (q[used] >> (6 - 2 * t)) & 3;
                        if (mode == 0) { cur[t + 1] = ZB_PREDEF; w->src_off[t + 1] = ZW_PREDEF; w->src_len[t + 1] = 0; }
                        else if (mode != 3) { cur[t + 1] = me; w->src_off[t + 1] = at0 + pos; w->src_len[t + 1] = bs; }
                        src[t] = (mode == 3) ? cur[t + 1] : (mode == 0 ? ZB_PREDEF : ZB_SELF);
                    }
                    B.ll_src = src[0]; B.of_src = src[1]; B.ml_src = src[2];
                }
            }
            B.comp_size = bs; B.regen_hint = lregen; B.nseq = nseq;
            B.seq_off = *scratch_used; *scratch_used += (((uint64_t)nseq * sizeof(ZDSeq)) + 15) & ~15ull;
            B.lit_off = *scratch_used; *scratch_used += ((uint64_t)lregen + 15) & ~15ull;
            pos += bs;
        }
        if (W) blocks_out[*nblocks_io] = B;
        (*nblocks_io)++;
        w->nblk++; walked++;
        if (last) break;
    }
    w->pos = at0 + pos;
    if (w->flags & ZF_CHECKSUM) { if (n - pos < 4) return ZMT_ST_TRUNCATED; pos += 4; }
    w->pos = at0 + pos;
    w->done = 1;
    *bound = bnd;
    return ZMT_ST_OK;
}

// Walks one zstd frame in frame[0..n) (frame header + 3-byte block headers + the two section headers of every
// compressed block).  `base_off` = offset of the frame's first byte in the decoder's input buffer.
// W = true writes one descriptor per accepted block at blocks_out[*nblocks_io++] (below index max_blocks); W = false
// only counts them.  Either way *nblocks_io advances by the block count, *scratch_used by the entropy scratch the
// blocks take (their seq_off / lit_off), *flags receives the ZF_* bits and, on success, *content_size the frame content
// size (the block bound without a content-size field).  *end = the frame's length on success, else the offset of the
// header element the walk stopped at.  Bytes behind the frame are the caller's business.  Returns ZMT_ST_*.
// The frame is one segment of zstd_walk_blocks that runs to its end.
// D, dict: as for zstd_walk_blocks.
template <bool W, bool D = false>
ZMT_HD int zstd_frame_walk(const uint8_t* frame, size_t n, uint64_t base_off, uint32_t frame_idx, ZBlk* blocks_out,
                           uint32_t* nblocks_io, uint32_t max_blocks, uint64_t* scratch_used, uint64_t* content_size,
                           uint32_t* flags, size_t* end, const zmt_zstd_dict_info* dict = nullptr)
{
    zmt_zstd_walk w = {};
    uint64_t bound = 0;
    const int r = zstd_walk_blocks<W, D>(frame, n, base_off, frame_idx, blocks_out, nblocks_io, max_blocks, scratch_used, &w,
                                         ~(size_t)0, ~0ull, &bound, dict);
    *flags = w.flags; *end = (size_t)w.pos;
    if (r == ZMT_ST_OK) *content_size = (w.flags & ZF_NO_SIZE) ? bound : w.content_size;
    return r;
}
