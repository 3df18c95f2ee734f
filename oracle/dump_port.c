/*
 * TEST INFRASTRUCTURE ONLY — our own C restatement of the MetOp X-band dump decoder (metop_dump_decoder):
 *   the module loop      plugins/noaa_metop_support/metop/module_metop_dump_decoder.cpp:41-79
 *   Correlator32 (QPSK)  src-core/common/codings/correlator32.cpp:3-64, 71-89, 134-176
 * with rotate_soft, the derandomiser and the interleaved Reed-Solomon decoder of oracle.c. Same C ABI as oracle/dump_harness.cpp (prefix
 * orc_); pinned to it by tests/test_metop_dump_oracle.py.
 *
 * The correlator's hard_buf is a 160 KiB buffer of which only the window's 1024 bytes are written; the rest is zero here, as the reference's
 * fresh allocation is (see dump_harness.cpp). The scan runs over bytes i < 8192 - 8, so it meets the window's tail mixed with zeros and
 * then the all-zero word.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "oracle.h"

#define F 8192
#define FRAME 1024
#define HARD_BUF (8192 * 20)

static uint32_t rotate_64(uint32_t word, int p)
{
    const uint32_t i = word & 0xaaaaaaaau, q = word & 0x55555555u;
    if (p == 1) word = ((i ^ 0xaaaaaaaau) >> 1) | (q << 1);
    else if (p == 2) word ^= 0xffffffffu;
    else if (p == 3) word = (i >> 1) | ((q ^ 0x55555555u) << 1);
    return ((word & 0x55555555u) << 1) | ((word & 0xaaaaaaaau) >> 1);
}
static uint32_t swap_iq(uint32_t w) { return ((w & 0xaaaaaaaau) >> 1) | ((w & 0x55555555u) << 1); }
static int corr_32(uint32_t a, uint32_t b) { return 32 - __builtin_popcount(a ^ b); }

typedef struct
{
    uint32_t sw[8];
    uint8_t *hard;          /* HARD_BUF bytes, zero behind the window */
    int8_t *pend;           /* soft bytes not consumed yet */
    long npend, cap_pend, base_off;
    int8_t buffer[2 * F];   /* the module's buffer; the second half stays zero */
} port_dump;

/* Correlator32::correlate for QPSK on F soft bytes: returns pos, sets phase, swap, cor */
static int correlate(port_dump *d, const int8_t *soft, int *phase, int *swap, int *cor)
{
    for (int i = 0; i < F / 8; i++) {
        uint8_t b = 0;
        for (int k = 0; k < 8; k++) b = (uint8_t)(b << 1 | (soft[8 * i + k] >= 0));
        d->hard[i] = b;
    }
    uint32_t cur = (uint32_t)d->hard[0] << 24 | (uint32_t)d->hard[1] << 16 | (uint32_t)d->hard[2] << 8 | d->hard[3];
    for (int p = 0; p < 8; p++) {
        const int c = corr_32(d->sw[p], cur);
        if (c > 27) { *cor = c; *phase = p % 4; *swap = p / 4 == 0; return 0; }
    }
    int best = 0, offset = 0, pos = 4;
    for (int i = 0; i < F - 8; i++) {
        for (int ii = 0; ii < 8; ii += 2) {
            for (int p = 0; p < 8; p++) {
                const int c = corr_32(d->sw[p], cur);
                if (c > best) { best = c; offset = i * 8 + ii; *phase = p % 4; *swap = p / 4 == 0; }
            }
            cur = cur << 2 | ((d->hard[pos] >> (6 - ii)) & 3);
        }
        pos++;
    }
    *cor = best;
    return offset;
}

void *orc_dump_create(void)
{
    port_dump *d = calloc(1, sizeof(port_dump));
    d->hard = calloc(HARD_BUF, 1);
    for (int p = 0; p < 4; p++) {
        d->sw[p] = rotate_64(0x1acffc1du, p);
        d->sw[4 + p] = rotate_64(swap_iq(0x1acffc1du) ^ 0xffffffffu, p);
    }
    return d;
}
void orc_dump_destroy(void *h)
{
    port_dump *d = h;
    free(d->hard);
    free(d->pend);
    free(d);
}

/* Same contract as ref_dump_run (dump_harness.cpp) */
long orc_dump_run(void *h, const int8_t *soft, long n, uint8_t *out, long cap_bytes, long *nbytes, long long *recs, long cap_frames)
{
    port_dump *d = h;
    if (d->npend + n > d->cap_pend) {
        d->cap_pend = 2 * (d->npend + n);
        d->pend = realloc(d->pend, d->cap_pend);
    }
    memcpy(d->pend + d->npend, soft, n);
    d->npend += n;
    const long size = d->npend;
    long o = 0, nf = 0, nb = 0;
    int8_t *buf = d->buffer;
    uint8_t frame[FRAME];
    while (size - o >= F) {
        memcpy(buf, d->pend + o, F);
        int phase = 0, swap = 0, cor = 0, errors[4] = {0, 0, 0, 0};
        const int pos = correlate(d, buf, &phase, &swap, &cor);
        const int shift = pos != 0 && pos < F;
        if (shift) {
            if (o + pos + F > size) break;
            memmove(buf, buf + pos, pos);
            memcpy(buf + F - pos, d->pend + o + F, pos);
        }
        if (nf >= cap_frames || nb + FRAME > cap_bytes) return -1;
        orc_rotate_soft(buf, F, phase, swap);
        for (int i = 0; i < FRAME; i++) {
            uint8_t b = 0;
            for (int y = 0; y < 8; y++) b = (uint8_t)(b << 1 | (buf[i * 8 + y] > 0));
            frame[i] = b ^ 0xFF;
        }
        orc_derand(frame + 4, FRAME - 4);
        orc_rs_decode_interleaved(frame + 4, 1, 4, 0, 0, errors);
        static const uint8_t sync[4] = {0x1a, 0xcf, 0xfc, 0x1d};
        memcpy(out + nb, sync, 4);
        memcpy(out + nb + 4, frame + 4, FRAME - 4);
        nb += FRAME;
        long long *rec = recs + 9 * nf;
        rec[0] = d->base_off + o + (shift ? pos : 0);
        rec[1] = pos;
        rec[2] = cor;
        rec[3] = phase;
        rec[4] = swap;
        for (int i = 0; i < 4; i++) rec[5 + i] = errors[i];
        nf++;
        o += F + (shift ? pos : 0);
    }
    memmove(d->pend, d->pend + o, size - o);
    d->npend = size - o;
    d->base_off += o;
    *nbytes = nb;
    return nf;
}
