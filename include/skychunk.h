/*
 * skychunk.h -- C ABI of the H100 chunk-processing stage (libskychunk.so).
 *
 * Drop-in boundary for the per-chunk hot path of Skyplane's gateway.  The reference has no FFI
 * (it is pure Python); these entry points replace, for one batch of chunks, the two calls
 *     data = lz4.frame.compress(data)          skyplane/gateway/operators/gateway_operator.py:358-361
 *     m = hashlib.md5(); m.update(b); digest   skyplane/obj_store/s3_interface.py:181-192
 * and hand back exactly what the sender needs for its wire header (gateway_operator.py:367-372):
 * the frame bytes, their length, and the 16-byte digest for Chunk.md5_hash (skyplane/chunk.py:21).
 *
 * Conventions: plain pointers and sizes, no exceptions, 0 = success / negative = error code.
 * The caller owns every host buffer; the library owns device memory, streams and events.
 * One sky_ctx per process per GPU; calls on one ctx are not thread-safe (the reference runs one
 * process per worker, gateway_operator.py:66-70).  A ctx must be created in the process that uses
 * it (after fork), never inherited.
 *
 * Output format: one LZ4 frame per chunk that lz4.frame.decompress (gateway_receiver.py:196)
 * restores bit-exactly: magic, FLG=0x68 (v01, independent blocks, content size), BD=0x40 (64 KiB),
 * u64le content size, header checksum, blocks (bit 31 set = stored raw), EndMark.  A zero-length
 * chunk yields the 11-byte frame liblz4 itself emits (content size omitted).  With SKY_F_CHECKSUM the
 * frame also carries LZ4's content checksum (FLG=0x6C, u32le XXH32 of the chunk after the EndMark), with
 * SKY_F_BLOCK_CHECKSUM a block checksum behind every block (FLG=0x78).
 * The receiver accepts block and content checksums in any frame and verifies them (SKY_D_CHECKSUM).
 */
#ifndef SKYCHUNK_H
#define SKYCHUNK_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define SKY_API __attribute__((visibility("default")))
#else
#define SKY_API
#endif

#define SKY_ABI_VERSION 4

/* error codes */
#define SKY_OK 0
#define SKY_E_INVALID (-1)   /* bad argument (null pointer, misaligned device pointer, n == 0 ...) */
#define SKY_E_NOGPU (-2)     /* no CUDA device / driver: there is NO CPU fallback */
#define SKY_E_CUDA (-3)      /* a CUDA call failed; see sky_last_error() */
#define SKY_E_CAPACITY (-4)  /* batch exceeds what the ctx was created for, dst_cap < sky_frame_bound(), or a chunk > 128 GiB */
#define SKY_E_BUSY (-5)      /* all slots hold un-waited tickets */
#define SKY_E_TICKET (-6)    /* unknown / already consumed ticket */
#define SKY_E_NOMEM (-7)
#define SKY_E_NOKEY (-8)     /* SKY_F_E2EE without sky_set_e2ee_key() / without nonces */

/* stage selection (0 = LZ4 + MD5).  SKY_F_MD5 alone is the reference's `compress: false` (gateway_daemon.py:235,
 * gateway_operator.py:358): the chunk is digested and passes through uncompressed. */
#define SKY_F_LZ4 1u
#define SKY_F_MD5 2u
/* end-to-end encryption behind the frame (sky_submit / sky_decode): every payload becomes PyNaCl's
 * SecretBox.encrypt() message  nonce(24) | tag(16) | ciphertext  (XSalsa20-Poly1305), as GatewaySender does with
 * e2ee_key_bytes (gateway_operator.py:183-186, :362-364) and the receiver undoes (gateway_receiver.py:191-193). */
#define SKY_F_E2EE 16u
#define SKY_BOX_OVERHEAD 40u
/* high-ratio frames (sky_submit, with or without SKY_F_E2EE, and sky_process_device): the same frame format, made by a
 * hash-chain match search with a lazy parse instead of the fast single-candidate parse.  Alone it means
 * LZ4 + MD5 + HC, as 0 means LZ4 + MD5; with stage bits it needs SKY_F_LZ4 (SKY_F_MD5 | SKY_F_HC is SKY_E_INVALID).
 * The digests come from the fused kernel's MD5-only mode running beside the HC kernel (two launches per batch). */
#define SKY_F_HC 32u
/* high-ratio level (python-lz4's compression_level, liblz4's hash-chain levels): bits 8..11 of flags hold a level
 * l in 3..9, and the search walks 2^(l-1) chain candidates per position -- more ratio for more GPU time.  A level field
 * of 0 with SKY_F_HC means level 5 (16 candidates), so SKY_F_HC_LEVEL(5) and SKY_F_HC make the same frames.  A level
 * field without SKY_F_HC, or outside 3..9, is SKY_E_INVALID.  The frame format does not depend on the level; the level
 * combines with SKY_F_CHECKSUM, SKY_F_E2EE and the stage bits as SKY_F_HC does.  sky_kernel_config(7) is the highest
 * level the library supports. */
#define SKY_F_HC_LEVEL(l) (SKY_F_HC | ((uint32_t)(l) << 8))
/* content checksum (sky_submit, with or without SKY_F_HC / SKY_F_E2EE, and sky_process_device): the frame carries
 * XXH32(chunk, seed 0) as LZ4's content checksum, so any LZ4 decoder (lz4.frame.decompress, liblz4) verifies that it
 * restores the chunk's bytes.  FLG becomes 0x6C (0x64 for an empty chunk, a 15-byte frame) and the frame ends with the
 * EndMark followed by u32le XXH32; out_len includes those 4 bytes, and dst_cap[i] >= sky_frame_bound(src_len[i]) + 4
 * (sky_box_bound(src_len[i]) + 4 with SKY_F_E2EE).  Alone it means LZ4 + MD5 + checksum; the MD5 lanes compute the
 * XXH32, so the digests always come back; without SKY_F_LZ4 (no frame to carry it) it is SKY_E_INVALID.  One more launch
 * per batch writes the checksums into the frames. */
#define SKY_F_CHECKSUM 64u
/* block checksums (sky_submit, with or without SKY_F_HC / SKY_F_HC_LEVEL, SKY_F_CHECKSUM and SKY_F_E2EE, and
 * sky_process_device): every block's data is followed by u32le XXH32(block data as stored in the frame, seed 0) -- the
 * compressed bytes, or the raw bytes of a stored block -- as liblz4 writes with blockChecksumFlag = 1, so any LZ4 decoder
 * (lz4.frame.decompress, liblz4, sky_decode) rejects a damaged block by its own checksum before decoding it.  FLG becomes
 * 0x78 (0x7C with SKY_F_CHECKSUM; 0x70 / 0x74 for an empty chunk, which has no block); the EndMark, the content checksum
 * and out_len move by 4 bytes per block, and dst_cap[i] >= sky_frame_bound(src_len[i]) + 4 * ceil(src_len[i] / 65536)
 * (+ 4 with SKY_F_CHECKSUM, + SKY_BOX_OVERHEAD with SKY_F_E2EE).  Alone it means LZ4 + MD5 + block checksums; without
 * SKY_F_LZ4 (no frame to carry them) it is SKY_E_INVALID.  The compressor CTA that writes a block hashes it; one more
 * launch per batch writes FLG and the header checksum byte. */
#define SKY_F_BLOCK_CHECKSUM 128u
/* frame verification (sky_submit, with any of the frame flags above and SKY_F_E2EE): before a batch's frames are sealed
 * or copied out, the GPU checks every frame against its chunk -- header exactly as the stage writes it, block words,
 * block and content checksums, and every block decoded against the chunk's bytes under liblz4's rules -- so that a frame
 * the stage returns restores its chunk under any LZ4 decoder.  A frame that fails is rewritten in place as the chunk's
 * stored-block frame (same header and checksum flags, every block stored raw; sky_frame_bound plus the checksum bytes,
 * which dst_cap already holds) and its status (sky_wait's verify[i]) is the failing check's SKY_D_* code.  Alone it means
 * LZ4 + MD5 + verify; without SKY_F_LZ4 (no frame) it is SKY_E_INVALID, and sky_process_device does not take it
 * (sky_verify_device runs the same check over frames in HBM).  Three more launches per batch.  It sits outside the
 * SKY_F_HC_LEVEL field. */
#define SKY_F_VERIFY 4096u
/* linked blocks (python-lz4's block_linked, liblz4's blockMode = linked), with SKY_F_HC / SKY_F_HC_LEVEL only (sky_submit,
 * sky_process_device, sky_verify_device): a match may reach up to 65535 bytes back, across its block's start into the
 * previous block of the chunk, which on text saves 9-17 % of the high-ratio mode's bytes.  FLG clears B.Indep (0x48,
 * 0x4C / 0x58 / 0x5C with the checksum flags) for a chunk of more than one block; a chunk of at most one block keeps the
 * independent FLG, as liblz4 writes it.  Every block is still made from the chunk's source bytes alone, so blocks compress
 * in parallel.  The receiver (sky_decode, lz4.frame.decompress) decodes a linked frame's blocks one after the other within
 * the chunk.  Without SKY_F_HC, or with SKY_F_MD5 alone, it is SKY_E_INVALID: the fast compressor has no linked mode, since its
 * parse would trail the reference's ratio even with the window.  sky_decode does not take it: a frame states its own block
 * mode. */
#define SKY_F_LINKED 8192u
/* optimal parse (sky_submit, sky_process_device, sky_verify_device), with SKY_F_HC / SKY_F_HC_LEVEL only, at any level and
 * with or without SKY_F_LINKED: the same match search, but instead of the lazy parse each block's sequences are chosen
 * by their cost in bytes (liblz4's optimal parse over the search's longest match per position, every shorter length at
 * the same offset priced as the sequence it makes).  The block is parsed in independent segments of
 * sky_kernel_config(8) bytes, which no match crosses, so that the segments are parsed in parallel.  The frame format is
 * unchanged, so any LZ4 decoder reads the frames; on Silesia-like data level 5 gains 1.3 % of ratio (1.7 % with
 * SKY_F_LINKED) for 3.8 % more GPU time.  Without SKY_F_HC, or with SKY_F_MD5 alone, it is SKY_E_INVALID.  For sky_verify_device it names the
 * compressor that made the frames, as SKY_F_HC does.  sky_decode does not take it: a frame states its own format. */
#define SKY_F_OPTIMAL 16384u
/* pass-through of incompressible chunks (sky_submit only): chunk i is sent as itself when its final frame -- after
 * SKY_F_VERIFY's repair, if that is set -- is not smaller than the chunk (frame_len[i] >= src_len[i]); every other chunk is
 * sent as its frame, byte for byte the frame the batch makes without this flag.  The frames are made as always; only what
 * comes back changes.  For a chunk that passes through: without SKY_F_E2EE out_len[i] = 0 and dst[i] is not written (as
 * with SKY_F_MD5 alone, the caller forwards its own input bytes, and nothing is copied back for it); with SKY_F_E2EE dst[i]
 * holds the SecretBox of the chunk's own bytes and out_len[i] = src_len[i] + SKY_BOX_OVERHEAD.  The digests always come
 * back, and SKY_F_VERIFY's statuses too.  sky_wait's compressed[i] says which payload each chunk got, and the ticket
 * needs it (see sky_wait).  It needs SKY_F_LZ4 (or no stage bit) and combines with SKY_F_HC / SKY_F_HC_LEVEL /
 * SKY_F_LINKED / SKY_F_OPTIMAL, SKY_F_E2EE and SKY_F_VERIFY.
 * With SKY_F_MD5 alone, SKY_F_CHECKSUM or SKY_F_BLOCK_CHECKSUM (a raw payload cannot carry the LZ4 checksums) it is
 * SKY_E_INVALID, as it is in sky_process_device, sky_verify_device and sky_decode: the receiver takes the chunks that pass
 * through as it takes SKY_F_MD5's payloads. */
#define SKY_F_PASSTHROUGH 32768u

typedef struct sky_ctx sky_ctx;

SKY_API const char *sky_strerror(int code);
SKY_API const char *sky_last_error(const sky_ctx *ctx); /* detail of the last SKY_E_CUDA on this ctx */
SKY_API int sky_abi_version(void);
SKY_API int sky_device_count(int *count);
/* PCI bus id ("0000:1b:00.0") of CUDA device `device` as the CUDA runtime orders devices (honours CUDA_VISIBLE_DEVICES,
 * unlike nvidia-smi -i); the host side maps it to the GPU's NUMA node before pinning staging memory. */
SKY_API int sky_device_pci_bus_id(int device, char *buf, int len);
/* Compile-time constants of the kernels in this build (tuning builds differ): what = 0 -> LZ4 match-table entries per
 * CTA, 1 -> warps per CTA of the fused kernel, 2 -> probe slots per segment, 3 -> log2 of the largest probe stride;
 * SKY_F_HC: 4 -> chain candidates searched per position at the default level (5), 5 -> log2 of the hash-head entries,
 * 6 -> length at which a position's search stops, 7 -> highest SKY_F_HC_LEVEL, 8 -> SKY_F_OPTIMAL's parse segment in bytes.
 * Unknown `what` returns 0 (so a library without SKY_F_HC reads 0 for 4..6, one without levels 0 for 7 and one without
 * SKY_F_OPTIMAL 0 for 8).  Parity tests feed
 * these to the sequential twins of the compressors (tools/lz4_tile_model.c, tools/lz4hc_model.c). */
SKY_API uint32_t sky_kernel_config(int what);

/* Worst-case frame bytes for an n-byte chunk: 15 + n + 4*ceil(n/65536) + 4 (11 when n == 0). */
SKY_API uint64_t sky_frame_bound(uint64_t n);

/* Create a context on `device` able to hold batches of up to max_chunks chunks totalling
 * max_batch_bytes input bytes.  n_slots >= 1 batches may be in flight through sky_submit at once
 * (each slot owns an input slab, an output slab and a stream); n_slots == 0 creates a ctx for
 * sky_process_device only (no slabs). */
SKY_API int sky_ctx_create(int device, uint64_t max_batch_bytes, uint32_t max_chunks, uint32_t n_slots, sky_ctx **out);
SKY_API int sky_ctx_destroy(sky_ctx *ctx);

/* Page-locked host memory for staging chunk bytes (cudaHostAlloc, portable). */
SKY_API void *sky_pinned_alloc(uint64_t bytes);
SKY_API int sky_pinned_free(void *p);

/* ---- host-buffer path (what GatewayOperator.process uses) -------------------------------------
 * sky_submit: asynchronously copies n chunks host->device, runs the fused kernel, and stages the
 *   per-chunk sizes and digests back.  src[i]/src_len[i] = chunk bytes; dst[i]/dst_cap[i] = where
 *   the frame goes (dst_cap[i] >= sky_frame_bound(src_len[i])).  All host buffers must stay valid
 *   until sky_wait returns.  Pinned buffers make the copies truly asynchronous.
 *   flags: SKY_F_* (0 = LZ4 + MD5, nonces may be NULL).  SKY_F_MD5 alone: digests only (dst / dst_cap may be NULL,
 *   out_len comes back 0: the caller forwards its own input bytes, is_compressed = False).  | SKY_F_E2EE: what comes
 *   back in dst[i] is the sealed box of the frame (or of the raw chunk when SKY_F_LZ4 is off), out_len[i] = its length
 *   = payload + SKY_BOX_OVERHEAD, dst_cap[i] >= sky_box_bound(src_len[i]); nonces = 24 bytes per chunk chosen by the
 *   caller (nacl.utils.random(24)).  The key is the ctx's (sky_set_e2ee_key; key32 = NULL switches E2EE off).
 * sky_wait: blocks until the batch is done, copies each frame device->host (exact length), and fills the outputs it is
 *   given, each optional: out_len[n], md5[16*n]; verify[n] = per chunk 0 (the frame restores the chunk) or the SKY_D_*
 *   code of the frame as the compressor made it, whose payload is now the stored-block frame (SKY_F_VERIFY);
 *   compressed[n] = per chunk 1 when its payload is a frame (or the SecretBox of a frame), 0 when it is the chunk itself
 *   (or the SecretBox of the chunk) -- WireProtocolHeader.is_compressed; without SKY_F_PASSTHROUGH it is 1 exactly when
 *   the ticket has SKY_F_LZ4.  kernel_ms = device time of the fused kernel.  Two requests are SKY_E_INVALID and leave the
 *   ticket waitable: verify != NULL on a ticket without SKY_F_VERIFY, and compressed == NULL on a SKY_F_PASSTHROUGH
 *   ticket (a caller that ignored the bit would label a sealed raw chunk as compressed). */
SKY_API int sky_submit(sky_ctx *ctx, uint32_t n, const void *const *src, const uint64_t *src_len, void *const *dst,
               const uint64_t *dst_cap, uint32_t flags, const uint8_t *nonces, uint64_t *ticket);
SKY_API int sky_wait(sky_ctx *ctx, uint64_t ticket, uint64_t *out_len, uint8_t *md5, int32_t *verify, uint8_t *compressed,
                     float *kernel_ms);
SKY_API int sky_set_e2ee_key(sky_ctx *ctx, const uint8_t *key32);
SKY_API uint64_t sky_box_bound(uint64_t n); /* sky_frame_bound(n) + SKY_BOX_OVERHEAD */

/* ---- device-resident path (kernel metric; inputs already in HBM) ------------------------------
 * Chunk i is d_src[src_off[i] .. +src_len[i]) ; its frame is written at d_dst + dst_off[i]
 * (capacity dst_cap[i] >= sky_frame_bound(src_len[i])).  src_off/dst_off must be multiples of 16
 * and both regions must be readable/writable up to the next multiple of 16.  `stream` is a
 * cudaStream_t (NULL = the ctx's own stream).  Synchronous: returns after the results are on the
 * host.  flags: SKY_F_* (0 = LZ4 + MD5). */
SKY_API int sky_process_device(sky_ctx *ctx, uint32_t n, const void *d_src, const uint64_t *src_off, const uint64_t *src_len,
                       void *d_dst, const uint64_t *dst_off, const uint64_t *dst_cap, uint32_t flags, void *stream,
                       uint64_t *out_len, uint8_t *md5, float *kernel_ms);

/* ---- receiver side: LZ4 frame decode + digest of the decoded bytes -----------------------------------
 * Replaces lz4.frame.decompress(to_write) (skyplane/gateway/operators/gateway_receiver.py:195-201) and supplies
 * the digest for the "# todo check hash" at gateway_receiver.py:231.  raw_len[i] is the expected decoded size
 * (WireProtocolHeader.raw_data_len, skyplane/chunk.py:100).  Accepts the frames this library emits (independent
 * 64 KiB blocks) and the reference sender's (linked blocks), with or without block and content checksums, which are
 * verified; status[i] = 0 or a SKY_D_* code (a bad frame is an
 * error status, never a crash); md5[16*i..] = MD5 of the decoded bytes.
 * sky_decode_device: frames and output already in HBM (out_off multiples of 16; each frame region must be readable
 * up to the next multiple of 4 bytes, each output region writable up to the next multiple of 16).  sky_decode: host
 * buffers, synchronous, through slot 0's slabs (needs n_slots >= 1).  Its flags are the stage bits the sender's
 * sky_submit was given, so every payload sky_submit makes has a receiver:
 *
 *     sky_submit flags                what is on the wire             sky_decode flags
 *     0 / SKY_F_LZ4 | SKY_F_MD5       LZ4 frame                       0 (or SKY_F_LZ4, SKY_F_LZ4 | SKY_F_MD5)
 *     ... | SKY_F_E2EE                SecretBox of the frame          SKY_F_E2EE (with or without the two bits)
 *     SKY_F_MD5 (`compress: false`)   the chunk's own bytes           SKY_F_MD5
 *     SKY_F_MD5 | SKY_F_E2EE          SecretBox of the chunk          SKY_F_MD5 | SKY_F_E2EE
 *     ... | SKY_F_PASSTHROUGH         per chunk, one of the rows      per chunk, by sky_wait's compressed[i]:
 *                                     above (frame or chunk)          the frames' row or the chunks' row
 *
 * SKY_F_E2EE: the payloads are sealed boxes, whose tags are checked and which are opened on the device first (status
 * SKY_D_AUTH for a forged / truncated box, whose bytes are never returned; SKY_E_NOKEY without a key).
 * SKY_F_MD5 alone: payload i IS chunk i (WireProtocolHeader.is_compressed = False): frames[i] / frame_len[i] are the
 * received bytes, raw_len[i] the header's raw_data_len; frame_len[i] != raw_len[i] is SKY_D_SIZE (the size check of
 * gateway_receiver.py:213-218).  The chunks are digested on the device by the launch sky_submit(SKY_F_MD5) makes and
 * nothing is copied back: dst may be NULL and a dst[i] is not written, as sky_submit(SKY_F_MD5) writes no dst.
 * SKY_F_MD5 | SKY_F_E2EE: every box is opened straight into the digest's input; the opened chunk is copied to dst[i]
 * (needed when raw_len[i] > 0).  An authentic box whose message is not raw_len[i] bytes long is SKY_D_SIZE and is not
 * copied out; SKY_D_AUTH comes before SKY_D_SIZE.  In both raw modes the digest of a chunk whose status is not 0 is 16 zero
 * bytes, and kernel_ms covers open + digest.  Any other flag bit is SKY_E_INVALID: a frame says itself which checksums
 * it carries and any compressor's frames decode alike, so the receiver has no frame option to take.
 * sky_decode_device takes no flags: for chunks already in HBM, receiving a raw chunk is sky_process_device(SKY_F_MD5). */
#define SKY_D_OK 0
#define SKY_D_BAD_HEADER (-1)
#define SKY_D_CORRUPT (-2)
#define SKY_D_SIZE (-3)
#define SKY_D_UNSUPPORTED (-4)
#define SKY_D_LAYOUT (-5)
#define SKY_D_TRUNCATED (-6)
#define SKY_D_AUTH (-7) /* SKY_F_E2EE: the box's Poly1305 tag does not verify (nacl.exceptions.CryptoError in the reference) */
#define SKY_D_CHECKSUM (-8) /* a block checksum or the content checksum (XXH32) does not match: lz4.frame.decompress raises */
#define SKY_D_MISMATCH (-9) /* SKY_F_VERIFY: the frame is well formed but decodes to other bytes than the chunk */
SKY_API int sky_decode_device(sky_ctx *ctx, uint32_t n, const void *d_frames, const uint64_t *frame_off, const uint64_t *frame_len,
                      void *d_out, const uint64_t *out_off, const uint64_t *raw_len, void *stream, int32_t *status, uint8_t *md5,
                      float *kernel_ms);
SKY_API int sky_decode(sky_ctx *ctx, uint32_t n, const void *const *frames, const uint64_t *frame_len, void *const *dst,
               const uint64_t *raw_len, uint32_t flags, int32_t *status, uint8_t *md5, float *kernel_ms);

/* ---- frame verification over frames in HBM (SKY_F_VERIFY's check and repair) -----------------------------------------
 * Chunk i is d_src[src_off[i] .. +src_len[i]) (d_src and src_off multiples of 16, readable up to the next multiple of 16),
 * its frame d_frames[frame_off[i] .. +frame_len[i]) (any alignment, readable up to the next multiple of 4 bytes).  flags:
 * the frame flags the frames were made with (SKY_F_CHECKSUM, SKY_F_BLOCK_CHECKSUM fix FLG and the trailer; the stage
 * and compressor bits are accepted as sky_submit takes them; SKY_F_E2EE or SKY_F_MD5 alone is SKY_E_INVALID).
 * content_xxh[i]: the chunk's XXH32, given exactly when SKY_F_CHECKSUM is set.  status[i] = 0 or the SKY_D_* code of the
 * check that failed.  frame_cap == NULL: check only, no byte changes.  Otherwise every failing frame is rewritten in place
 * as its stored-block frame, frame_len[i] becomes its length, and nothing outside [frame, frame + frame_cap[i]) is written;
 * frame_cap[i] < sky_frame_bound(src_len[i]) + the flags' checksum bytes is SKY_E_CAPACITY.  Synchronous; kernel_ms =
 * device time of the check (and repair).  Uses slot 0's metadata, as sky_process_device does. */
SKY_API int sky_verify_device(sky_ctx *ctx, uint32_t n, const void *d_src, const uint64_t *src_off, const uint64_t *src_len, void *d_frames,
                      const uint64_t *frame_off, uint64_t *frame_len, const uint64_t *frame_cap, const uint32_t *content_xxh,
                      uint32_t flags, void *stream, int32_t *status, float *kernel_ms);

/* Device-memory helpers so a host without torch can drive the device path. */
SKY_API int sky_device_alloc(sky_ctx *ctx, uint64_t bytes, void **dptr);
SKY_API int sky_device_free(sky_ctx *ctx, void *dptr);
SKY_API int sky_memcpy_h2d(sky_ctx *ctx, void *dptr, const void *host, uint64_t bytes);
SKY_API int sky_memcpy_d2h(sky_ctx *ctx, void *host, const void *dptr, uint64_t bytes);

/* Number of kernel launches issued through this ctx so far (bench.py's gpu_launches). */
SKY_API uint64_t sky_launch_count(const sky_ctx *ctx);

#ifdef __cplusplus
}
#endif
#endif /* SKYCHUNK_H */
