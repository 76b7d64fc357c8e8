/* TEST INFRASTRUCTURE ONLY.
 *
 * A stand-in for the five libdeflate calls the reference's PNG writer makes (src/timg-png.cc), so that the
 * reference's own canvases can be compiled and run without libdeflate (which is not part of its tree).  The
 * "compressor" writes the zlib stream with STORED deflate blocks, laid out exactly as timg_b200/csrc/png.cu does:
 *   78 01 | per block of <= 65535 bytes: BFINAL/BTYPE=00 byte, LEN, NLEN (little-endian) and the bytes | Adler-32
 *   (big-endian); the last block has BFINAL set; an empty input is one empty final block.
 * The compression level is ignored.  Checksums come from zlib (-lz).
 * With this header on the include path, the reference's code produces the whole framed kitty / iTerm2 stream
 * (Sub filter, chunk CRCs, base64, chunking, headers) for the PNG bytes this library produces. */
#ifndef ORACLE_DEFLATE_STORED_LIBDEFLATE_H
#define ORACLE_DEFLATE_STORED_LIBDEFLATE_H

#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <zlib.h>

#ifdef __cplusplus
extern "C" {
#endif

struct libdeflate_compressor {
    int level;
};

static inline struct libdeflate_compressor *libdeflate_alloc_compressor(int compression_level) {
    struct libdeflate_compressor *c = (struct libdeflate_compressor *)malloc(sizeof(struct libdeflate_compressor));
    if (c) c->level = compression_level;
    return c;
}

static inline void libdeflate_free_compressor(struct libdeflate_compressor *c) { free(c); }

static inline size_t libdeflate_zlib_compress_bound(struct libdeflate_compressor *c, size_t in_nbytes) {
    (void)c;
    const size_t blocks = in_nbytes ? (in_nbytes + 65534) / 65535 : 1;
    return 2 + 5 * blocks + in_nbytes + 4;
}

/* Returns the bytes written, or 0 if they do not fit (libdeflate's convention). */
static inline size_t libdeflate_zlib_compress(struct libdeflate_compressor *c, const void *in, size_t in_nbytes, void *out,
                                              size_t out_nbytes_avail) {
    const size_t need = libdeflate_zlib_compress_bound(c, in_nbytes);
    if (need > out_nbytes_avail) return 0;
    const uint8_t *src = (const uint8_t *)in;
    uint8_t *o = (uint8_t *)out;
    *o++ = 0x78;
    *o++ = 0x01;
    size_t left = in_nbytes;
    do {
        const size_t len = left < 65535 ? left : 65535;
        *o++ = left == len ? 1 : 0;
        *o++ = (uint8_t)len;
        *o++ = (uint8_t)(len >> 8);
        *o++ = (uint8_t)~len;
        *o++ = (uint8_t)(~len >> 8);
        for (size_t i = 0; i < len; ++i) *o++ = src[i];
        src += len;
        left -= len;
    } while (left);
    const uint32_t a = (uint32_t)adler32(adler32(0L, Z_NULL, 0), (const Bytef *)in, (uInt)in_nbytes);
    *o++ = (uint8_t)(a >> 24);
    *o++ = (uint8_t)(a >> 16);
    *o++ = (uint8_t)(a >> 8);
    *o++ = (uint8_t)a;
    return (size_t)(o - (uint8_t *)out);
}

static inline uint32_t libdeflate_crc32(uint32_t crc, const void *buffer, size_t len) {
    return (uint32_t)crc32((uLong)crc, (const Bytef *)buffer, (uInt)len);
}

#ifdef __cplusplus
}
#endif
#endif /* ORACLE_DEFLATE_STORED_LIBDEFLATE_H */
