/* TEST INFRASTRUCTURE ONLY.
 *
 * A stand-in for the five libdeflate calls the reference's PNG writer makes (src/timg-png.cc) that REPLAYS a zlib
 * stream: libdeflate_zlib_compress ignores its level and writes the stream that oracle_replay_stream() (defined by
 * the program, e.g. the door oracle/ref_graphics_replay.cc) gives for its input, the filtered scanlines.  The input is
 * passed so that a program whose canvases encode on several threads can pick each frame's stream by its content.  The bound is the stored-block size, which
 * no stream of this library exceeds.  Checksums come from zlib (-lz).
 * With this header on the include path, the reference's own png::Encode writes the PNG chunks, lengths and CRCs, and
 * its canvases the base64, chunking, headers and placeholders, around a deflate stream this library produced. */
#ifndef ORACLE_DEFLATE_REPLAY_LIBDEFLATE_H
#define ORACLE_DEFLATE_REPLAY_LIBDEFLATE_H

#include <stddef.h>
#include <stdint.h>
#include <string.h>
#include <zlib.h>

#ifdef __cplusplus
extern "C" {
#endif

/* defined by the program: the zlib stream libdeflate_zlib_compress returns for the scanlines in[0, in_nbytes), and its
 * length */
const uint8_t *oracle_replay_stream(const void *in, size_t in_nbytes, size_t *n);

struct libdeflate_compressor {
    int level;
};

static inline struct libdeflate_compressor *libdeflate_alloc_compressor(int compression_level) {
    static struct libdeflate_compressor c;
    c.level = compression_level;
    return &c;
}

static inline void libdeflate_free_compressor(struct libdeflate_compressor *c) { (void)c; }

static inline size_t libdeflate_zlib_compress_bound(struct libdeflate_compressor *c, size_t in_nbytes) {
    (void)c;
    const size_t blocks = in_nbytes ? (in_nbytes + 65534) / 65535 : 1;
    return 2 + 5 * blocks + in_nbytes + 4;
}

/* Returns the bytes written, or 0 if they do not fit (libdeflate's convention). */
static inline size_t libdeflate_zlib_compress(struct libdeflate_compressor *c, const void *in, size_t in_nbytes, void *out,
                                              size_t out_nbytes_avail) {
    (void)c;
    size_t n = 0;
    const uint8_t *s = oracle_replay_stream(in, in_nbytes, &n);
    if (n > out_nbytes_avail) return 0;
    memcpy(out, s, n);
    return n;
}

static inline uint32_t libdeflate_crc32(uint32_t crc, const void *buffer, size_t len) {
    return (uint32_t)crc32((uLong)crc, (const Bytef *)buffer, (uInt)len);
}

#ifdef __cplusplus
}
#endif
#endif /* ORACLE_DEFLATE_REPLAY_LIBDEFLATE_H */
