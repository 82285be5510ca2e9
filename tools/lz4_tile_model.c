/*
 * lz4_tile_model.c -- sequential CPU twin of the round-2 GPU block compressor (skyplane_b200/csrc/lz4.cuh).
 *
 * NOT the reference's algorithm (that is oracle/skyoracle.c) and NOT product code: a development tool.  It replays the
 * kernel's parse on the host, byte for byte, so (a) design options can be compared for compression ratio without a GPU
 * (tools/tile_study.py) and (b) the GPU output can be diffed against a sequential implementation of the same rules
 * (tests/test_tools_model.py, tests/test_gpu_parity.py::test_frames_equal_sequential_twin).
 *
 * The parse, per 64 KiB block (the kernel runs it with one CTA per block: a prober warp and several parser warps):
 *   segment = seg_slots probe slots, slot i at position seg_pos + (i << slog); segments tile the block back to back.
 *             slog starts at 0 for the first two segments; segment s+2's slog is 0 if segment s had any hit, else segment
 *             s+1's slog plus one (up to max_step_log) -- one segment of delay, so the kernel's two prober warps never
 *             wait for each other's verdict.
 *   probe   = 32 slots (a group) at a time: hash 5 bytes, look the table entry (pos16 | tag16) up; hit = tag equal and
 *             entry older than the slot.  A slot whose full 32-bit hash equals that of the slot 3, 4 or 8 places before it
 *             in the same group takes that one as its candidate instead (short periods: pixels, words, doubles -- the
 *             table cannot know them yet).  Then the group's slots replace their table entries, the last one staying.
 *             No byte of the candidate is read here.
 *   parse   = per segment, independently of every other segment: cursor and anchor start at the segment start; walk the
 *             hits at or after the cursor; measure the real match length from byte 0 (this is also the verification),
 *             clipped to the segment end (and to the block's last-5-bytes rule); drop it if < 4; extend backwards by up
 *             to 8 bytes but not past the anchor; record the sequence; cursor = anchor = match end.
 *   emit    = the block's sequences are the segments' sequences in order; literals a segment leaves behind its last match
 *             (or a whole segment without a match) are carried into the next sequence.  Standard LZ4 block format.
 *             A block whose compressed size would exceed L-1 is stored raw (return 0), as LZ4F_makeBlock does.
 *   linked  = (study mode, tile_compress_block_linked; the kernel does not implement it) blocks j >= 1 of a chunk may
 *             match into the previous 64 KiB window, FLG B.Indep clear (for chunks of more than one block, see
 *             tools/tile_model.py).  The table starts seeded from that window instead of empty: its positions
 *             65536 - seed .. 65531 inserted in order, last writer wins (what sequential insertion leaves behind),
 *             each as (pos16 | tag16) with pos16 relative to the previous block.  A probe's candidate offset is
 *             (p - pos16) mod 65536: an entry above p is in the previous window at offset p + 65536 - pos16, one below p
 *             is in this block (a seeded entry below p is read as a position of this block: the parse verifies every
 *             candidate, so such a stale entry only costs a probe).  Offset 0 is no hit.  Nothing else changes: the
 *             parse verifies and extends against the chunk's source bytes (backward extension may cross the block
 *             start), and block j depends on source bytes only, never on block j-1's compressed output.  Block 0 of a
 *             chunk is the independent block.
 *
 * Build: gcc -O2 -shared -fPIC -o tools/bin/liblz4tile.so tools/lz4_tile_model.c
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define MINMATCH 4
#define MFLIMIT 12
#define LASTLITERALS 5

typedef struct {
    int entries;       /* table entries (kernel: 4096; index = mulhi(hash, entries)) */
    int seg_slots;     /* probe slots per segment (kernel: 1024) */
    int max_step_log;  /* largest probe stride = 1 << this (kernel: 4) */
    int back_ext;      /* 1 = extend accepted matches backwards by up to 8 bytes (kernel: 1) */
    int clip;          /* 1 = matches end at the segment end (kernel: 1; 0 shows what the segment independence costs) */
    int group_lag;     /* 1 = the 32 slots of a group all look the table up before any of them is inserted (kernel: 1);
                          0 = every slot sees the slots before it (study variant: what a fully sequential probe would find) */
    int near_mask;     /* with group_lag: bit d-1 set = a slot also compares its 5-byte hash with the slot d places before it
                          in its group; the nearest equal one is its candidate, ahead of the table's (kernel: 0x8c = 3, 4, 8) */
} tile_opts;

static uint32_t rd32(const uint8_t *p) { uint32_t v; memcpy(&v, p, 4); return v; }

static uint32_t emit(uint8_t *out, uint32_t op, const uint8_t *src, uint32_t anchor, uint32_t ll, uint32_t ml, uint32_t off) {
    uint32_t mcode = ml ? ml - MINMATCH : 0;
    out[op++] = (uint8_t)(((ll < 15 ? ll : 15) << 4) | (mcode < 15 ? mcode : 15));
    if (ll >= 15) { uint32_t r = ll - 15; for (; r >= 255; r -= 255) out[op++] = 255; out[op++] = (uint8_t)r; }
    memcpy(out + op, src + anchor, ll); op += ll;
    if (ml) {
        out[op++] = (uint8_t)off; out[op++] = (uint8_t)(off >> 8);
        if (mcode >= 15) { uint32_t r = mcode - 15; for (; r >= 255; r -= 255) out[op++] = 255; out[op++] = (uint8_t)r; }
    }
    return op;
}

static uint32_t hash5(const uint8_t *p) { return rd32(p) * 2654435761u + p[4] * 0x85EBCA6Bu; }  /* 5 bytes, two 32-bit multiplies */
static uint32_t hidx(uint32_t hf, const tile_opts *o) { return (uint32_t)(((uint64_t)hf * (uint32_t)o->entries) >> 32); }
static uint32_t htag(uint32_t hf) { return (hf >> 8) & 0xffffu; }  /* hash bytes 1-2: one PRMT in the kernel */

typedef struct { uint64_t probes, hits, accepted, segments; } tile_stats;
static tile_stats g_stats;
void tile_model_stats(tile_stats *s, int reset) { *s = g_stats; if (reset) memset(&g_stats, 0, sizeof g_stats); }

/* returns compressed size, or 0 if the block does not shrink (store raw); out capacity >= L + 2048.
   prefix = bytes of the previous window readable before src (0: an independent block; linked: 65536 for blocks j >= 1),
   seed = how many of its last positions seed the table (linked only). */
static uint32_t compress_block(const uint8_t *src, uint32_t L, uint8_t *out, const tile_opts *o, uint32_t prefix, uint32_t seed) {
    const uint32_t S = (uint32_t)o->seg_slots, limit = L - 1;
    uint32_t *tab = calloc((size_t)o->entries, 4);  /* pos | tag << 16 ; 0 = (pos 0, tag 0) = "empty" */
    if (prefix)  /* linked: the previous window's positions q (hash inside the window), in order, the last one staying */
        for (uint32_t q = prefix - seed; q + 5 <= prefix; q++) {
            const uint32_t hf = hash5(src - prefix + q);
            tab[hidx(hf, o)] = q | (htag(hf) << 16);
        }
    uint16_t *off = malloc(2 * S);
    uint8_t *hit = malloc(S);
    uint32_t anchor = 0 /* start of the literals not yet emitted */, op = 0, result = 0;
    uint32_t ghf[32];
    if (L >= MFLIMIT + 1) {
        const uint32_t mflimit = L - MFLIMIT, matchlimit = L - LASTLITERALS;
        uint32_t seg_pos = 0, slog = 0, slog_next = 0;  /* slog of this segment / of the next one */
        while (seg_pos <= mflimit) {
            g_stats.segments++;
            /* ---- probe, one group of 32 slots at a time */
            int anyhit = 0;
            for (uint32_t g = 0; g < S; g += 32) {
                for (uint32_t i = g; i < g + 32; i++) {
                    const uint32_t p = seg_pos + (i << slog);
                    hit[i] = 0;
                    ghf[i - g] = 0;
                    if (p > mflimit) continue;
                    const uint32_t hf = hash5(src + p);
                    const uint32_t e = tab[hidx(hf, o)], epos = e & 0xffffu;
                    ghf[i - g] = hf;
                    g_stats.probes++;
                    if (prefix) {  /* linked: offset (p - pos16) mod 65536, 0 = no hit */
                        if ((e >> 16) == htag(hf) && ((p - epos) & 0xffffu)) { hit[i] = 1; off[i] = (uint16_t)(p - epos); }
                    } else if ((e >> 16) == htag(hf) && epos < p) { hit[i] = 1; off[i] = (uint16_t)(p - epos); }
                    if (o->group_lag) {  /* an equal hash 3, 4 or 8 slots back in the group is the nearer candidate */
                        for (uint32_t d = 1; d <= i - g; d++)
                            if ((((uint32_t)o->near_mask >> (d - 1)) & 1u) && ghf[i - g - d] == hf) { hit[i] = 1; off[i] = (uint16_t)(d << slog); break; }
                    } else tab[hidx(hf, o)] = p | (htag(hf) << 16);
                    if (hit[i]) { anyhit = 1; g_stats.hits++; }
                }
                if (o->group_lag)  /* the group's slots replace the table entries in slot order (the last one stays) */
                    for (uint32_t i = g; i < g + 32; i++) {
                        const uint32_t p = seg_pos + (i << slog);
                        if (p <= mflimit) tab[hidx(ghf[i - g], o)] = p | (htag(ghf[i - g]) << 16);
                    }
            }
            /* ---- parse: depends on nothing outside this segment */
            const uint32_t seg_lim = seg_pos + (S << slog);  /* first byte of the next segment */
            const uint32_t mlim = (o->clip && seg_lim < matchlimit) ? seg_lim : matchlimit;
            uint32_t cur = seg_pos, lanchor = seg_pos;  /* local cursor / anchor */
            if (!o->clip && anchor > seg_pos) cur = lanchor = anchor;  /* (study variant: one parse across segments) */
            for (uint32_t i = 0; i < S; i++) {
                if (!hit[i]) continue;
                uint32_t pos = seg_pos + (i << slog);
                if (pos < cur || pos >= mlim) continue;
                int64_t cand = (int64_t)pos - off[i];  /* < 0: in the previous window (linked) */
                const uint32_t maxlen = mlim - pos;
                uint32_t mlen = 0;
                while (mlen < maxlen && src[pos + mlen] == src[cand + mlen]) mlen++;
                if (mlen < MINMATCH) continue;
                if (o->back_ext) {
                    uint32_t room = pos - lanchor;
                    if (cand + prefix < room) room = (uint32_t)(cand + prefix);
                    if (room > 8) room = 8;
                    uint32_t b = 0;
                    while (b < room && src[pos - 1 - b] == src[cand - 1 - b]) b++;
                    pos -= b; cand -= b; mlen += b;
                }
                op = emit(out, op, src, anchor, pos - anchor, mlen, (uint32_t)(pos - cand));
                anchor = cur = lanchor = pos + mlen;
                g_stats.accepted++;
                if (op > L + 1024) goto done;  /* (model only) hopeless and about to overrun the caller's buffer */
            }
            seg_pos = seg_lim;
            {   /* this segment's verdict decides the stride two segments on */
                const uint32_t after = anyhit ? 0 : (slog_next < (uint32_t)o->max_step_log ? slog_next + 1 : slog_next);
                slog = slog_next;
                slog_next = after;
            }
        }
    }
    if (L - anchor + (L - anchor) / 255 + 2 + op <= L + 2040) op = emit(out, op, src, anchor, L - anchor, 0, 0);
    else op = L;  /* cannot fit anyway */
    if (op <= limit) result = op;
done:
    free(tab); free(off); free(hit);
    return result;
}

uint32_t tile_compress_block(const uint8_t *src, uint32_t L, uint8_t *out, const tile_opts *o) {
    return compress_block(src, L, out, o, 0, 0);
}

/* block j >= 1 of a linked chunk: src[-65536 .. -1] is block j-1; seed = its last positions that seed the table */
uint32_t tile_compress_block_linked(const uint8_t *src, uint32_t L, uint8_t *out, const tile_opts *o, uint32_t seed) {
    return compress_block(src, L, out, o, 65536, seed);
}
