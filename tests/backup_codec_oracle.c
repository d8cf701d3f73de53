/*
 * backup_codec_oracle.c -- codec.DecodeToBuffer and codec.EncodeFromBuffer (codec/codec.go:402-414, 456-467) restated
 * one decision at a time on the CPU oracle's Decoder and Encoder (oracle/oracle.c), with encoding/binary's PutUvarint
 * and Uvarint.  TEST INFRASTRUCTURE ONLY: the checker of dgx_decode_to_buffer_rows and dgx_encode_from_buffer_rows in
 * tests/ and smoke(), and the CPU legs of tools/bench_ops.py C11; backup_codec_oracle.py compiles it together with
 * oracle/oracle.c into a temporary directory.
 *
 * orc_put_uvarint(buf, x)               binary.PutUvarint: little-endian groups of 7 bits, high bit = more follows
 * orc_uvarint(buf, len, &n)             binary.Uvarint: n > 0 bytes read; n == 0 buffer ends inside the value; n < 0
 *                                       overflow (an 11th byte, or a 10th byte > 1)
 * orc_decode_to_buffer(p, out)          DecodeToBuffer: out must hold 10 * ExactLen bytes; returns the bytes written
 * orc_encode_from_buffer(buf, len, bs, &pack)
 *                                       EncodeFromBuffer: 0 and the pack (NULL: the nil pack); -1 where the reference
 *                                       panics (n < 0: buf[n:] with a negative index), -2 where it loops forever
 *                                       (n == 0: buf never shrinks)
 */
#include <stdlib.h>
#include <string.h>

#include "../oracle/oracle.h"

size_t orc_put_uvarint(uint8_t* buf, uint64_t x);
uint64_t orc_uvarint(const uint8_t* buf, size_t len, long* n);
size_t orc_decode_to_buffer(const orc_pack* p, uint8_t* out);
int orc_encode_from_buffer(const uint8_t* buf, size_t len, int block_size, orc_pack** out);

size_t orc_put_uvarint(uint8_t* buf, uint64_t x) {
    size_t i = 0;
    while (x >= 0x80) {
        buf[i] = (uint8_t)x | 0x80;
        x >>= 7;
        i++;
    }
    buf[i] = (uint8_t)x;
    return i + 1;
}

uint64_t orc_uvarint(const uint8_t* buf, size_t len, long* n) {
    uint64_t x = 0;
    unsigned s = 0;
    for (size_t i = 0; i < len; i++) {
        if (i == 10) { /* MaxVarintLen64: overflow */
            *n = -(long)(i + 1);
            return 0;
        }
        uint8_t b = buf[i];
        if (b < 0x80) {
            if (i == 9 && b > 1) { /* overflow */
                *n = -(long)(i + 1);
                return 0;
            }
            *n = (long)(i + 1);
            return x | (uint64_t)b << s;
        }
        x |= (uint64_t)(b & 0x7f) << s;
        s += 7;
    }
    *n = 0;
    return 0;
}

size_t orc_decode_to_buffer(const orc_pack* p, uint8_t* out) {
    uint64_t last = 0;
    size_t o = 0, len = 0;
    orc_decoder* dec = orc_decoder_new(p);
    for (const uint64_t* uids = orc_decoder_seek(dec, 0, ORC_SEEK_START, &len); len > 0;
         uids = orc_decoder_next(dec, &len)) {
        for (size_t i = 0; i < len; i++) {
            o += orc_put_uvarint(out + o, uids[i] - last);
            last = uids[i];
        }
    }
    orc_decoder_free(dec);
    return o;
}

int orc_encode_from_buffer(const uint8_t* buf, size_t len, int block_size, orc_pack** out) {
    /* Encode is Encoder.Add for every uid, then Done (codec.go:393-399): the uids are collected and handed to it */
    uint64_t* uids = (uint64_t*)malloc((len + 1) * sizeof(uint64_t));
    size_t nu = 0;
    uint64_t prev = 0;
    while (len > 0) {
        long n;
        uint64_t uid = orc_uvarint(buf, len, &n);
        if (n <= 0) {
            free(uids);
            *out = NULL;
            return n < 0 ? -1 : -2;
        }
        buf += n;
        len -= (size_t)n;
        uint64_t next = prev + uid;
        uids[nu++] = next;
        prev = next;
    }
    *out = orc_encode(uids, nu, block_size);
    free(uids);
    return 0;
}
