/*
 * TEST INFRASTRUCTURE ONLY — never linked into or called from the product path.
 *
 * Our own C restatement of ccsds_turbo_decoder (CCSDSTurboDecoderModule::process, module_ccsds_turbo_decoder.cpp:137-235), with
 * CCSDSTurbo::decode (ccsds_turbo.cpp:156-198), turbo_decode (libturbocodes.c:137-201) and convcode_extrinsic (libconvcodes.c:355-549)
 * written from their description: the same operations in the same order, in double, each rounded on its own (built with
 * -ffp-contract=off). tests/test_turbo_oracle.py pins it bit for bit to the reference (oracle/_ref/libsatref_turbo.so) where that was
 * built, and to tests/golden/turbo_pins.json everywhere. Same C ABI as oracle/turbo_harness.cpp with the prefix orc_ instead of ref_.
 *
 * The module's buffer after a shift by pos is memmove(buf, buf + pos, pos) followed by pos new bytes at its end; for pos > F / 2 that
 * memmove reads past the F-byte buffer, here a buffer of 2F bytes whose second half is zero.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define STATES 16
#define MEM 4

typedef struct
{
    int comps;
    int next[STATES][2], prev[STATES][2], prev_u[STATES][2];
    int out[STATES][2][4];
} code_t;

/* recursive systematic code, feedback "0011", feed-forward taps fwd[c] (tap 0 on the new first register, taps 1..4 on registers 1..4 =
   state bits 3..0); the predecessors of each state in the order: states ascending, input 0 before input 1 */
static void make_code(code_t *c, const char *const *fwd, int comps)
{
    int filled[STATES] = {0};
    c->comps = comps;
    for (int st = 0; st < STATES; st++)
        for (int u = 0; u < 2; u++) {
            const int first = u ^ ((st >> 1) & 1) ^ (st & 1); /* registers 3 and 4 */
            const int ns = (st >> 1) | (first << (MEM - 1));
            for (int k = 0; k < comps; k++) {
                int o = (fwd[k][0] - '0') & first;
                for (int i = 0; i < MEM; i++)
                    o ^= (fwd[k][i + 1] - '0') & ((st >> (MEM - 1 - i)) & 1);
                c->out[st][u][k] = o;
            }
            c->next[st][u] = ns;
            c->prev[ns][filled[ns]] = st;
            c->prev_u[ns][filled[ns]] = u;
            filled[ns]++;
        }
}

static void codes_of(int rate, code_t *upper, code_t *lower)
{
    static const char *u2[] = {"10011", "11011"}, *u4[] = {"10011", "10101", "11111"}, *u6[] = {"10011", "11011", "10101", "11111"};
    static const char *l1[] = {"11011"}, *l6[] = {"11011", "11111"};
    if (rate == 6) {
        make_code(upper, u6, 4);
        make_code(lower, l6, 2);
    } else {
        make_code(upper, rate == 4 ? u4 : u2, rate == 4 ? 3 : 2);
        make_code(lower, l1, 1);
    }
}

static void interleaver(int base, int *pi)
{
    static const int p[8] = {31, 37, 43, 47, 53, 59, 61, 67};
    const int K = 8 * base;
    for (int s = 0; s < K; s++) {
        const int m = s % 2, i = s / (2 * base), j = s / 2 - i * base, t = (19 * i + 1) % 4, q = t % 8;
        const int c = (p[q] * j + 21 * m) % base;
        pi[s] = 2 * (t + c * 4 + 1) - m - 1;
    }
}

static double exp_sum(double a, double b)
{
    const double d = a - b;
    if (a > b)
        return a;
    return b + log(1 + exp(-d > 0 ? d : -d));
}

/* -g / (2 nv), g = sum over the components of (rho_j - (2 out_j - 1))^2 */
static double branch(const double *rho, const int *out, int comps, double nv)
{
    double g = 0;
    for (int j = 0; j < comps; j++) {
        const double x = rho[j] - (2 * out[j] - 1);
        g += x * x;
    }
    return -g / (2 * nv);
}

/* One component pass on rx (comps x (K + 4) values): app0 / app1 (K values) are replaced by the extrinsic values; dec != NULL: the
   decisions one > zero */
static void extrinsic(const double *rx, int K, double *app0, double *app1, const code_t *c, double nv, int *dec)
{
    const int N = K + MEM, C = c->comps;
    const double T = 1e10;
    double *ap = malloc(sizeof(double) * 2 * N), *bw = malloc(sizeof(double) * N * STATES), *fw = malloc(sizeof(double) * N * STATES);
    double *ext = malloc(sizeof(double) * 2 * N);
    for (int i = 0; i < N; i++) {
        ap[i] = i < K ? app0[i] : log(0.5);
        ap[N + i] = i < K ? app1[i] : log(0.5);
    }
    for (int s = 0; s < STATES; s++)
        bw[(N - 1) * STATES + s] = s ? -T : 0;
    for (int i = N - 2; i >= 0; i--) {
        const double *rho = rx + C * (i + 1);
        double *row = bw + i * STATES, mx;
        for (int s = 0; s < STATES; s++) {
            double B = -T;
            for (int u = 0; u < 2; u++)
                B = exp_sum(B, ap[u * N + i + 1] + bw[(i + 1) * STATES + c->next[s][u]] + branch(rho, c->out[s][u], C, nv));
            row[s] = B;
        }
        mx = row[0];
        for (int s = 0; s < STATES; s++)
            mx = row[s] > mx ? row[s] : mx;
        for (int s = 0; s < STATES; s++)
            row[s] -= mx;
    }
    for (int s = 0; s < STATES; s++)
        fw[s] = s ? -T : 0;
    for (int i = 1; i < N; i++) {
        const double *rho = rx + C * (i - 1);
        double *row = fw + i * STATES, mx;
        for (int s = 0; s < STATES; s++) {
            double F = -T;
            for (int n = 0; n < 2; n++) {
                const int st = c->prev[s][n], in = c->prev_u[s][n];
                F = exp_sum(F, ap[in * N + i - 1] + fw[(i - 1) * STATES + st] + branch(rho, c->out[st][in], C, nv));
            }
            row[s] = F;
        }
        mx = row[0];
        for (int s = 0; s < STATES; s++)
            mx = row[s] > mx ? row[s] : mx;
        for (int s = 0; s < STATES; s++)
            row[s] -= mx;
    }
    for (int i = 0; i < N; i++) {
        const double *rho = rx + C * i;
        for (int u = 0; u < 2; u++) {
            double E = -T;
            for (int s = 0; s < STATES; s++)
                E = exp_sum(E, fw[i * STATES + s] + bw[i * STATES + c->next[s][u]] + branch(rho, c->out[s][u], C, nv));
            ext[u * N + i] = E;
        }
        if (i < K) {
            app0[i] = ext[i];
            app1[i] = ext[N + i];
        }
    }
    if (dec)
        for (int i = 0; i < K; i++)
            dec[i] = ap[N + i] + ext[N + i] > ap[i] + ext[i];
    free(ap);
    free(bw);
    free(fw);
    free(ext);
}

static int asm_bits_of(int rate) { return rate == 2 ? 64 : (rate == 3 ? 96 : (rate == 4 ? 128 : 192)); }
static int codeword_of(int rate, int base) { return (rate == 2 ? 2 : rate) * (8 * base + MEM); }

/* the decoder of one frame: cw floats (after the sign fix) -> base bytes */
static void decode(int rate, int base, int iters, const int *pi, const code_t *up, const code_t *lo, const float *in, uint8_t *outb)
{
    const int K = 8 * base, N = K + MEM, cb = up->comps + lo->comps;
    const float sigma = 0.707f;
    const double nv = sigma * sigma;
    double *rx = calloc((size_t)cb * N, sizeof(double)), *su = malloc(sizeof(double) * up->comps * N), *sl = malloc(sizeof(double) * lo->comps * N);
    double *m0 = malloc(sizeof(double) * K), *m1 = malloc(sizeof(double) * K), *l0 = malloc(sizeof(double) * K), *l1 = malloc(sizeof(double) * K);
    int *dec = malloc(sizeof(int) * K);
    if (rate == 2) /* block b of 3 keeps position 0, and position 1 (even b) or 2 (odd b) */
        for (int b = 0, j = 0; b < N; b++) {
            rx[3 * b] = in[j++];
            rx[3 * b + (b & 1 ? 2 : 1)] = in[j++];
        }
    else
        for (int k = 0; k < cb * N; k++)
            rx[k] = in[k];
    for (int b = 0; b < N; b++) {
        for (int j = 0; j < up->comps; j++)
            su[b * up->comps + j] = rx[b * cb + j];
        for (int j = 0; j < lo->comps; j++)
            sl[b * lo->comps + j] = rx[b * cb + up->comps + j];
    }
    for (int i = 0; i < K; i++)
        m0[i] = m1[i] = log(0.5);
    for (int it = 0; it < iters; it++) {
        extrinsic(su, K, m0, m1, up, nv, NULL);
        for (int i = 0; i < K; i++) {
            l0[i] = m0[pi[i]];
            l1[i] = m1[pi[i]];
        }
        extrinsic(sl, K, l0, l1, lo, nv, it == iters - 1 ? dec : NULL);
        for (int i = 0; i < K; i++) {
            m0[pi[i]] = l0[i];
            m1[pi[i]] = l1[i];
        }
    }
    memset(outb, 0, base);
    for (int i = 0; i < K; i++)
        if (dec[i])
            outb[pi[i] / 8] |= 0x80 >> (pi[i] % 8);
    free(rx); free(su); free(sl); free(m0); free(m1); free(l0); free(l1); free(dec);
}

static unsigned crc16(const uint8_t *d, int n)
{
    unsigned crc = 0xFFFF;
    for (int t = 0; t < n; t++) {
        crc ^= (unsigned)d[t] << 8;
        for (int k = 0; k < 8; k++)
            crc = (crc & 0x8000 ? (crc << 1) ^ 0x1021 : crc << 1) & 0xFFFF;
    }
    return crc;
}

typedef struct
{
    int rate, base, iters, A, cw, F;
    float table[192];
    unsigned char pn[255];
    int *pi;
    code_t up, lo;
    int8_t *pend, *buf;
    long npend, cap, base_off;
    float *fl;
} orc_turbo;

void *orc_turbo_create(int rate, int base, int iters)
{
    static const char *hex[] = {"034776C7272895B0", "25D5C0CE8990F6C9461BF79C", "034776C7272895B0FCB88938D8D76A4F",
                                "25D5C0CE8990F6C9461BF79CDA2A3F31766F0936B9E40863"};
    orc_turbo *t = calloc(1, sizeof(orc_turbo));
    const char *h = hex[rate == 2 ? 0 : (rate == 3 ? 1 : (rate == 4 ? 2 : 3))];
    t->rate = rate;
    t->base = base;
    t->iters = iters;
    t->A = asm_bits_of(rate);
    t->cw = codeword_of(rate, base);
    t->F = t->cw + t->A;
    for (int i = 0; i < t->A; i++) {
        const char c = h[i / 4];
        const int nib = c <= '9' ? c - '0' : c - 'A' + 10;
        t->table[i] = (nib >> (3 - i % 4)) & 1 ? 1.0f : -1.0f;
    }
    uint8_t reg = 0xFF;
    for (int i = 0; i < 255; i++) {
        t->pn[i] = reg >> 7;
        reg = (uint8_t)((reg << 1) | (((reg >> 7) ^ (reg >> 4) ^ (reg >> 2) ^ reg) & 1));
    }
    t->pi = malloc(sizeof(int) * 8 * base);
    interleaver(base, t->pi);
    codes_of(rate, &t->up, &t->lo);
    t->buf = calloc(2 * (size_t)t->F, 1);
    t->fl = malloc(sizeof(float) * t->F);
    return t;
}

void orc_turbo_destroy(void *h)
{
    orc_turbo *t = h;
    free(t->pi); free(t->pend); free(t->buf); free(t->fl); free(t);
}

int orc_turbo_frame_size(void *h) { return ((orc_turbo *)h)->F; }

/* see ref_turbo_run (oracle/turbo_harness.cpp) */
long orc_turbo_run(void *h, const int8_t *soft, long n, uint8_t *out, long cap_bytes, long *nbytes, long long *recs, long cap_frames)
{
    orc_turbo *t = h;
    if (t->npend + n > t->cap) {
        t->cap = t->npend + n;
        t->pend = realloc(t->pend, t->cap);
    }
    memcpy(t->pend + t->npend, soft, n);
    t->npend += n;
    const int F = t->F, A = t->A;
    long o = 0, nf = 0, nb = 0;
    uint8_t frame[1119];
    while (t->npend - o >= F) {
        memcpy(t->buf, t->pend + o, F);
        for (int i = 0; i < F; i++)
            t->fl[i] = (float)t->buf[i] / 127.0f;
        int pos = 0, swapped = 0;
        float best = 0;
        for (int p = 0; p < F - A; p++) {
            float acc = 0.0f;
            for (int k = 0; k < A; k++)
                acc += t->fl[p + k] * t->table[k];
            if (acc > best) { best = acc; pos = p; swapped = 0; }
            if (-acc > best) { best = -acc; pos = p; swapped = 1; }
        }
        if (pos != 0) {
            if (o + pos + F > t->npend)
                break;
            memmove(t->buf, t->buf + pos, pos);
            memcpy(t->buf + F - pos, t->pend + o + F, pos);
        }
        if (nf >= cap_frames)
            return -1;
        for (int c = 0; c < t->cw; c++)
            if (t->pn[c % 255])
                t->buf[A + c] = ~t->buf[A + c];
        for (int i = 0; i < F; i++) {
            const float x = (float)t->buf[i] / 127.0f;
            t->fl[i] = swapped ? -x : x;
        }
        decode(t->rate, t->base, t->iters, t->pi, &t->up, &t->lo, t->fl + A, frame + 4);
        frame[0] = 0x1a; frame[1] = 0xcf; frame[2] = 0xfc; frame[3] = 0x1d;
        const int ok = crc16(frame + 4, t->base - 2) == ((unsigned)frame[t->base + 2] << 8 | frame[t->base + 3]);
        if (ok) {
            if (nb + t->base + 4 > cap_bytes)
                return -1;
            memcpy(out + nb, frame, t->base + 4);
            nb += t->base + 4;
        }
        long long *rec = recs + 6 * nf;
        uint32_t cbits;
        memcpy(&cbits, &best, 4);
        rec[0] = t->base_off + o + pos;
        rec[1] = pos;
        rec[2] = cbits;
        rec[3] = swapped;
        rec[4] = ok;
        rec[5] = pos == 0;
        nf++;
        o += pos + F;
    }
    memmove(t->pend, t->pend + o, t->npend - o);
    t->npend -= o;
    t->base_off += o;
    *nbytes = nb;
    return nf;
}

int orc_turbo_perm(int base, int *out)
{
    interleaver(base, out);
    return 8 * base;
}

/* see ref_turbo_half (oracle/turbo_harness.cpp) */
void orc_turbo_half(int rate, int base, int lower, const double *stream, double *app0, double *app1, int decision, int *decoded)
{
    code_t up, lo;
    codes_of(rate, &up, &lo);
    const float sigma = 0.707f;
    extrinsic(stream, 8 * base, app0, app1, lower ? &lo : &up, sigma * sigma, decision ? decoded : NULL);
}
