/*
 * TEST INFRASTRUCTURE ONLY — the CPU oracle ("port") of the CCSDS LDPC decoder (ccsds_ldpc_decoder, rate 7/8 C2 code).
 *
 * A from-scratch C restatement of what CCSDSLDPCDecoderModule::process (module_ccsds_ldpc_decoder.cpp:134-277) computes with the
 * generic decoder, with and without internal_stream (BPSK_CCSDS_Deframer, bpsk_ccsds_deframer.cpp:24-122), so that the tests have a
 * checker where oracle/_ref is absent. tests/test_ldpc_oracle.py pins it bit for bit to the reference's own code
 * (oracle/_ref/libsatref_ldpc.so) and, without it, to the digests of tests/golden/ldpc_pins.json (tests/golden/make_ldpc_pins.py). Same C ABI as ldpc_harness.cpp with the prefix orc_.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../satdump_b200/csrc/ldpc_c2_table.inc"

#define ROWS (LDPC_C2_BY * LDPC_C2_CIRC) /* 1022 */
#define VNS (LDPC_C2_BX * LDPC_C2_CIRC)  /* 8176 */
#define DEG (2 * LDPC_C2_BX)             /* 32, every row */
#define ASM_BITS 32
#define CW 8160
#define F (CW + ASM_BITS)

/* the CCSDS pseudo-random sequence, one bit per entry (LFSR h(x) = x^8+x^7+x^5+x^3+1 from all ones; period 255) */
static uint8_t pn_bit[255];
static void build_pn(void)
{
    uint8_t reg = 0xFF;
    for (int i = 0; i < 255; i++) {
        pn_bit[i] = reg >> 7;
        const uint8_t nb = ((reg >> 7) ^ (reg >> 4) ^ (reg >> 2) ^ reg) & 1;
        reg = (uint8_t)((reg << 1) | nb);
    }
}

/* H row by row, columns ascending (make_ccsds.cpp:407-430 adds row block 0's 511 rows, then row block 1's) */
static int H[ROWS][DEG];
static int h_ready = 0;
static void build_h(void)
{
    if (h_ready)
        return;
    for (int y = 0; y < LDPC_C2_BY; y++)
        for (int r = 0; r < LDPC_C2_CIRC; r++) {
            int *row = H[y * LDPC_C2_CIRC + r];
            for (int x = 0; x < LDPC_C2_BX; x++) {
                int a = (ldpc_c2_offsets[y][x][0] + r) % LDPC_C2_CIRC, b = (ldpc_c2_offsets[y][x][1] + r) % LDPC_C2_CIRC;
                if (a > b) { int t = a; a = b; b = t; }
                row[2 * x] = LDPC_C2_CIRC * x + a;
                row[2 * x + 1] = LDPC_C2_CIRC * x + b;
            }
        }
    h_ready = 1;
}

/* LDPCDecoderGeneric::decode (ldpc_decoder_generic.cpp:69-194): layered min-sum over int16 variable nodes, check nodes 0..1021 in turn.
   A check node's outgoing magnitude is the smallest |incoming| of the other edges (min1, or min2 at the edges equal to min1), both
   capped at 255; its sign is the parity of the other edges' signs. Returns the number of info positions (< 7154) whose hard decision
   differs from the sign of the input. */
static int16_t vns[VNS];
static int16_t c2v[ROWS][DEG];
static int decode_cw(const int8_t *in /* VNS */, uint8_t *out /* VNS */, int it)
{
    build_h();
    for (int i = 0; i < VNS; i++)
        vns[i] = in[i];
    memset(c2v, 0, sizeof(c2v));
    while (it--)
        for (int r = 0; r < ROWS; r++) {
            int16_t m[DEG];
            int neg = 0, min1 = 255, min2 = 255;
            for (int k = 0; k < DEG; k++) {
                m[k] = (int16_t)(vns[H[r][k]] - c2v[r][k]);
                neg ^= m[k] < 0;
                const int a = abs(m[k]);
                if (a < min1) { min2 = min1; min1 = a; }
                else if (a < min2) min2 = a;
            }
            for (int k = 0; k < DEG; k++) {
                const int mag = abs(m[k]) == min1 ? min2 : min1;
                const int16_t msg = (int16_t)((neg ^ (m[k] < 0)) ? -mag : mag);
                c2v[r][k] = msg;
                vns[H[r][k]] = (int16_t)(m[k] + msg);
            }
        }
    int corr = 0;
    for (int i = 0; i < VNS; i++) {
        out[i] = vns[i] >= 0;
        if (i < VNS - ROWS && (out[i] > 0) != (in[i] > 0))
            corr++;
    }
    return corr;
}

/* BPSK_CCSDS_Deframer (bpsk_ccsds_deframer.cpp:24-122): bit-serial ASM search; NOSYNC (2) exact match of the ASM or its inverse, SYNCING (6)
   fewer than 6 differing bits, SYNCED after more than 10 good ASMs (12) fewer than 12; frames of size bits start with the ASM itself */
typedef struct
{
    int size, state, in_frame, inversion, bit, good, invalid;
    uint32_t sync, shifter;
    uint8_t *buf;
} Deframer;
static void defr_reset_frame(Deframer *d)
{
    memset(d->buf, 0, d->size / 8);
    for (int k = 0; k < 4; k++)
        d->buf[k] = (uint8_t)(d->sync >> (24 - 8 * k));
    d->bit = 32;
}
static int defr_work(Deframer *d, const uint8_t *in, int n, uint8_t *out)
{
    int nf = 0;
    for (int i = 0; i < n; i++) {
        d->shifter = d->shifter << 1 | in[i];
        if (d->in_frame) {
            const uint8_t b = in[i] ^ (uint8_t)d->inversion;
            d->buf[d->bit / 8] = (uint8_t)(d->buf[d->bit / 8] << 1 | b);
            d->bit++;
            if (d->bit == d->size)
                memcpy(out + (size_t)nf++ * (d->size / 8), d->buf, d->size / 8);
            else if (d->bit == d->size + 31)
                d->in_frame = 0;
            continue;
        }
        const uint32_t want = d->inversion ? ~d->sync : d->sync;
        const int diff = __builtin_popcount(d->shifter ^ want);
        if (d->state == 2) {
            if (d->shifter == d->sync || d->shifter == ~d->sync) {
                d->inversion = d->shifter != d->sync;
                defr_reset_frame(d);
                d->in_frame = 1;
                d->state = 6;
                d->good = d->invalid = 0;
            }
        } else if (d->state == 6) {
            if (diff < d->state) {
                defr_reset_frame(d);
                d->in_frame = 1;
                d->invalid = 0;
                if (++d->good > 10)
                    d->state = 12;
            } else {
                d->invalid++;
                d->good = 0;
                if (d->invalid > 2)
                    d->state = 2;
            }
        } else {
            if (diff < d->state) {
                defr_reset_frame(d);
                d->in_frame = 1;
            } else {
                d->good = d->invalid = 0;
                d->state = 2;
            }
        }
    }
    return nf;
}

typedef struct
{
    Deframer *defr; /* internal_stream */
    int constellation, iterations, derandomize, nsync;
    float sync[4][ASM_BITS];
    int8_t *pend;
    long npend, cap, base;
    uint8_t out[CW]; /* ldpc_output_buffer: bits 8158 / 8159 never written (0) */
} Ldpc;

/* ---- CorrelatorGeneric (generic_correlator.cpp:7-64, 137-149, 176-263) for the 32-bit ASM 0x1ACFFC1D */
static void modulate(float *buf, const uint8_t *bits)
{
    for (int i = 0; i < ASM_BITS; i++)
        buf[i] = bits[i] ? 1.0f : -1.0f;
}
static void rotate_buf(float *buf, float deg)
{
    const float ph = deg * 0.01745329; /* computed in double, stored as float */
    const float c = cosf(ph), s = sinf(ph);
    for (int i = 0; i < ASM_BITS / 2; i++) {
        const float re = buf[2 * i], im = buf[2 * i + 1];
        buf[2 * i] = (re * c) - (im * s);
        buf[2 * i + 1] = (im * c) + (re * s);
    }
}
static void make_syncwords(Ldpc *d)
{
    uint8_t bits[ASM_BITS];
    for (int i = 0; i < ASM_BITS; i++)
        bits[i] = (0x1acffc1du >> (31 - i)) & 1;
    if (d->constellation == 0) {
        d->nsync = 2;
        modulate(d->sync[0], bits);
        modulate(d->sync[1], bits);
        rotate_buf(d->sync[1], 180);
    } else if (d->constellation == 1) {
        d->nsync = 4;
        for (int s = 0; s < 4; s++) {
            modulate(d->sync[s], bits);
            if (s)
                rotate_buf(d->sync[s], 90.0f * s);
        }
    } else {
        d->nsync = 4;
        modulate(d->sync[0], bits);
        modulate(d->sync[1], bits);
        uint8_t last = 0; /* Q delayed by one symbol: the syncword as seen when the wrong rail was delayed */
        for (int i = 0; i < ASM_BITS / 2; i++) {
            const uint8_t back = bits[2 * i + 1];
            bits[2 * i + 1] = last;
            last = back;
        }
        modulate(d->sync[2], bits);
        modulate(d->sync[3], bits);
        rotate_buf(d->sync[0], 90);
        rotate_buf(d->sync[1], 270);
        rotate_buf(d->sync[3], 180);
    }
}

/* best position in [0, F - 32): the first maximum of the fp32 scores if it is > 0, else 0 */
static int correlate(const Ldpc *d, const int8_t *soft, int *best_sync, float *cor)
{
    float conv[F];
    for (int i = 0; i < F; i++)
        conv[i] = ((float)soft[i]) / 63.0f; /* volk_8i_s32f_convert_32f(.., 127 / 2, ..) */
    float best = 0;
    int pos = 0, bs = 0;
    for (int i = 0; i < F - ASM_BITS; i++)
        for (int s = 0; s < d->nsync; s++) {
            float acc = 0.0f;
            for (int k = 0; k < ASM_BITS; k++)
                acc += conv[i + k] * d->sync[s][k];
            if (acc > best) {
                best = acc;
                bs = s;
                pos = i;
            }
        }
    *best_sync = bs;
    *cor = best;
    return pos;
}

/* rotate_soft (rotation.cpp:4-63) */
static void rotate_soft(int8_t *s, int n, int phase, int swap)
{
    for (int i = 0; i < n; i++)
        if (s[i] == -128)
            s[i] = -127;
    if (swap)
        for (int i = 0; i < n; i += 2) {
            const int8_t t = s[i + 1];
            s[i + 1] = s[i];
            s[i] = t;
        }
    for (int i = 0; i < n; i += (phase == 2 ? 1 : 2)) {
        if (phase == 1) { const int8_t t = s[i]; s[i] = s[i + 1]; s[i + 1] = -t; }
        else if (phase == 2) s[i] = -s[i];
        else if (phase == 3) { const int8_t t = s[i]; s[i] = -s[i + 1]; s[i + 1] = t; }
    }
}

void *orc_ldpc_create(int constellation, int iterations, int derandomize, int internal_cadu_size, unsigned internal_asm)
{
    Ldpc *d = calloc(1, sizeof(Ldpc));
    if (internal_cadu_size > 0) {
        d->defr = calloc(1, sizeof(Deframer));
        d->defr->size = internal_cadu_size;
        d->defr->sync = internal_asm;
        d->defr->state = 2;
        d->defr->buf = calloc(internal_cadu_size / 8 + 8, 1);
    }
    d->constellation = constellation;
    d->iterations = iterations;
    d->derandomize = derandomize;
    make_syncwords(d);
    build_h();
    build_pn();
    return d;
}
void orc_ldpc_destroy(void *h)
{
    Ldpc *d = h;
    if (d->defr) {
        free(d->defr->buf);
        free(d->defr);
    }
    free(d->pend);
    free(d);
}

long orc_ldpc_run(void *h, const int8_t *soft, long n, uint8_t *out, long cap_bytes, long *nbytes, long long *recs, long cap_frames)
{
    Ldpc *d = h;
    if (d->npend + n > d->cap) {
        d->cap = (d->npend + n) * 2;
        d->pend = realloc(d->pend, d->cap);
    }
    memcpy(d->pend + d->npend, soft, n);
    d->npend += n;
    long o = 0, nf = 0, nb = 0;
    int8_t sb[F], cw[VNS];
    while (d->npend - o >= F) {
        int best;
        float cor;
        const int pos = correlate(d, d->pend + o, &best, &cor);
        if (pos != 0 && o + pos + F > d->npend)
            break;
        if (nf >= cap_frames)
            return -1;
        memcpy(sb, d->pend + o + pos, F);
        int phase = 0, swap = 0; /* generic_correlator.cpp:233-262 */
        if (d->constellation == 0) phase = best ? 2 : 0;
        else if (d->constellation == 1) phase = best;
        else { static const int ph[4] = {1, 3, 0, 2}; phase = ph[best]; swap = best / 2; }
        if (d->constellation == 2) { /* module_ccsds_ldpc_decoder.cpp:159-173: re-delay Q, the last Q becomes 0 */
            rotate_soft(sb, F, phase, 0);
            if (swap) {
                for (int i = 0; i < F / 2 - 1; i++)
                    sb[2 * i + 1] = sb[2 * i + 3];
                sb[F - 1] = 0;
            }
        } else
            rotate_soft(sb, F, phase, swap);
        if (d->derandomize) /* derand_ccsds_soft: invert where the 255-bit PN sequence has a one */
            for (int i = 0; i < CW; i++)
                if (pn_bit[i % 255])
                    sb[ASM_BITS + i] = ~sb[ASM_BITS + i];
        /* CCSDSLDPC::decode (ccsds_ldpc.cpp:76-123): 18 zero (shortened) positions, then 8158 soft bytes */
        memset(cw, 0, 18);
        memcpy(cw + 18, sb + ASM_BITS, VNS - 18);
        uint8_t full[VNS];
        const int corr = decode_cw(cw, full, d->iterations);
        memcpy(d->out, full + 18, VNS - 18);
        int defr_state = 0;
        if (d->defr) { /* the first 7136 decoded bits through the deframer (:233-242) */
            static uint8_t tmp[2][F];
            const int fb = d->defr->size / 8;
            uint8_t *fr = fb * 2 <= (int)sizeof(tmp) ? tmp[0] : malloc((size_t)fb * 2);
            const int k = defr_work(d->defr, d->out, VNS - ROWS - 18, fr);
            if (nb + (long)k * fb > cap_bytes)
                return -1;
            memcpy(out + nb, fr, (size_t)k * fb);
            nb += (long)k * fb;
            if (fr != tmp[0])
                free(fr);
            defr_state = d->defr->state;
        } else {
            if (nb + 1024 > cap_bytes)
                return -1;
            uint8_t *dst = out + nb;
            const uint32_t sync = 0x1acffc1du;
            memcpy(dst, &sync, 4); /* host byte order (:252-256) */
            for (int b = 0; b < CW / 8; b++) {
                uint8_t v = 0;
                for (int k = 0; k < 8; k++)
                    v = (uint8_t)(v << 1 | d->out[8 * b + k]);
                dst[4 + b] = v;
            }
            nb += 1024;
        }
        long long *rec = recs + 8 * nf;
        uint32_t cbits;
        memcpy(&cbits, &cor, 4);
        rec[0] = d->base + o + pos;
        rec[1] = pos;
        rec[2] = cbits;
        rec[3] = phase;
        rec[4] = swap;
        rec[5] = corr;
        rec[6] = pos == 0;
        rec[7] = defr_state;
        nf++;
        o += pos + F;
    }
    memmove(d->pend, d->pend + o, d->npend - o);
    d->npend -= o;
    d->base += o;
    *nbytes = nb;
    return nf;
}

int orc_ldpc_decode(void *h, const int8_t *codeword, uint8_t *out, int iterations)
{
    (void)h;
    int8_t cw[VNS];
    uint8_t full[VNS];
    memset(cw, 0, 18);
    memcpy(cw + 18, codeword, VNS - 18);
    const int corr = decode_cw(cw, full, iterations);
    memcpy(out, full + 18, VNS - 18);
    return corr;
}

int orc_ldpc_matrix(int *cols, int cap_rows)
{
    if (cap_rows < ROWS)
        return -1;
    build_h();
    memcpy(cols, H, sizeof(H));
    return ROWS;
}
