/*
 * tests/bc6h_oracle_encode.c -- TEST INFRASTRUCTURE ONLY (never linked into libhap_b200.so).
 *
 * The oracle of the library's BC6H encoder (hap_b200/csrc/bc6h_encode.cuh), written apart from it.  It is built on the
 * decoder oracle (tests/bc6h_oracle.c, included whole): the same per-mode field lists, partition table, unquantisation and
 * final scale, so its blocks are packed and scored by the format as the oracle restates it, not as the kernel does.
 * Exports bc6h_oracle_encode besides the decoder oracle's functions.  Built by tests/bc6h_encode_util.py; checked in
 * tests/test_bc6h_encode_cpu.py.  Layouts: RGBA16F (R, G, B, A binary16) row-major, 4*w values per row; blocks row-major
 * over (w/4) x (h/4).
 */
#include <math.h>

#include "bc6h_oracle.c"

/* ---- the oracle encoder ----------------------------------------------------------------------------------------------
 * RGBA16F -> BC6H, sequential and exhaustive: every one of the 14 modes, every one of the 32 partitions of the two-region
 * modes.  Per (mode, partition): each region's endpoints start at its two texels farthest apart, then two rounds of
 * least-squares endpoints (a double-precision 2x2 solve per channel, in the integer domain the decoder interpolates in)
 * with the indices of the round before.  The best block of each mode is then improved by +-1 nudges of each quantised
 * endpoint component until no nudge lowers the error.  Every error is the exact one: endpoints unquantised and
 * interpolated as the decoder above does, each texel given its best index, the squared differences of the decoded and
 * source sign-magnitude integers summed over R, G and B.  A transformed mode whose deltas do not fit their bits after the
 * wrap is not a candidate.  Input rules: UF16 takes negatives, -0 and NaN as 0 and +Inf as 0x7BFF; SF16 takes NaN as 0,
 * +-Inf as +-0x7BFF and -0 as +0. */

static int src_value(uint16_t h, int is_signed)
{
    int mag = h & 0x7FFF;
    if (mag > 0x7C00) mag = 0;
    else if (mag == 0x7C00) mag = 0x7BFF;
    if (!(h & 0x8000)) return mag;
    return is_signed ? -mag : 0;
}

static int half_value(uint16_t h) { return (h & 0x8000) ? -(h & 0x7FFF) : h; }

/* the interpolated value of least magnitude that finish() maps to x */
static int target_of(int x, int is_signed)
{
    const int a = x < 0 ? -x : x;
    int v = a * (is_signed ? 32 : 64) / 31;
    while (finish(v, is_signed) < a) v++;
    while (v > 0 && finish(v - 1, is_signed) >= a) v--;
    return x < 0 ? -v : v;
}

static int q_lo(int prec, int is_signed) { return is_signed ? -(prec >= 16 ? 32767 : (1 << (prec - 1)) - 1) : 0; }
static int q_hi(int prec, int is_signed) { return is_signed ? (prec >= 16 ? 32767 : (1 << (prec - 1)) - 1) : (prec >= 16 ? 65535 : (1 << prec) - 1); }

/* the code of `prec` bits whose unquantised value is nearest v */
static int quantize_nearest(double v, int prec, int is_signed)
{
    const int lo = q_lo(prec, is_signed), hi = q_hi(prec, is_signed);
    const double scale = is_signed ? (prec >= 16 ? 1.0 : (double)(1 << (prec - 1)) / 32768.0) : (prec >= 16 ? 1.0 : (double)(1 << prec) / 65536.0);
    int q0 = (int)floor(v * scale), best = lo;
    double bd = 1e30;
    for (int q = q0 - 1; q <= q0 + 1; q++) {
        int qq = q < lo ? lo : q > hi ? hi : q;
        double d = fabs(unquantize(qq, prec, is_signed) - v);
        if (d < bd) { bd = d; best = qq; }
    }
    return best;
}

typedef struct {
    uint64_t err;
    int mode, partition, valid;
    int q[4][3];      /* quantised endpoints a0 b0 a1 b1 in the order stored */
    int idx[16];
} oracle_cand;

/* exact error of the quantised endpoints c->q in mode m, partition c->partition: every texel's best index; then the
 * anchors made to fit by swapping endpoints and mirroring indices, and the deltas checked */
static void oracle_eval(const int src[16][3], int is_signed, oracle_cand *c)
{
    const bc6h_mode *m = &bc6h_modes[c->mode];
    const int two = m->regions == 2, ib = two ? 3 : 4, levels = 1 << ib;
    int ep[4][3];
    for (int e = 0; e < 4; e++)
        for (int k = 0; k < 3; k++) ep[e][k] = unquantize(c->q[e][k], m->prec, is_signed);
    c->err = 0;
    for (int t = 0; t < 16; t++) {
        const int s = two ? bc6h_part[c->partition][t] : 0;
        uint64_t be = UINT64_MAX;
        for (int i = 0; i < levels; i++) {
            const int w = ib == 3 ? bc6h_w3[i] : bc6h_w4[i];
            uint64_t e = 0;
            for (int k = 0; k < 3; k++) {
                const int v = half_value(finish((ep[2 * s][k] * (64 - w) + ep[2 * s + 1][k] * w + 32) >> 6, is_signed));
                const int64_t d = v - src[t][k];
                e += (uint64_t)(d * d);
            }
            if (e < be) { be = e; c->idx[t] = i; }
        }
        c->err += be;
    }
    for (int s = 0; s < (two ? 2 : 1); s++) {
        const int at = s == 0 ? 0 : bc6h_anchor[c->partition];
        if (c->idx[at] < levels / 2) continue;
        for (int t = 0; t < 16; t++)
            if ((two ? bc6h_part[c->partition][t] : 0) == s) c->idx[t] = levels - 1 - c->idx[t];
        for (int k = 0; k < 3; k++) { int x = c->q[2 * s][k]; c->q[2 * s][k] = c->q[2 * s + 1][k]; c->q[2 * s + 1][k] = x; }
    }
    c->valid = 1;
    if (m->transformed)
        for (int e = 1; e < 2 * m->regions; e++)
            for (int k = 0; k < 3; k++) {
                const int d = sign_extend((c->q[e][k] - c->q[0][k]) & ((1 << m->prec) - 1), m->prec);
                if (d < -(1 << (m->delta[k] - 1)) || d > (1 << (m->delta[k] - 1)) - 1) c->valid = 0;
            }
}

static int better(const oracle_cand *a, const oracle_cand *b) { return a->valid && (!b->valid || a->err < b->err); }

/* least-squares endpoints of region s with the indices of c; 0 when every texel of the region has one weight */
static int oracle_lsq(const int src[16][3], int is_signed, const oracle_cand *c, int s, double a[3], double b[3])
{
    const int two = bc6h_modes[c->mode].regions == 2;
    double aa = 0, ab = 0, bb = 0, ax[3] = {0, 0, 0}, bx[3] = {0, 0, 0};
    for (int t = 0; t < 16; t++) {
        if ((two ? bc6h_part[c->partition][t] : 0) != s) continue;
        const double w = (two ? bc6h_w3[c->idx[t]] : bc6h_w4[c->idx[t]]) / 64.0, v = 1.0 - w;
        aa += v * v; ab += v * w; bb += w * w;
        for (int k = 0; k < 3; k++) {
            const double y = src[t][k] * (is_signed ? 32.0 : 64.0) / 31.0;
            ax[k] += v * y; bx[k] += w * y;
        }
    }
    const double det = aa * bb - ab * ab;
    if (det < 1e-9) return 0;
    for (int k = 0; k < 3; k++) {
        a[k] = (bb * ax[k] - ab * bx[k]) / det;
        b[k] = (aa * bx[k] - ab * ax[k]) / det;
    }
    return 1;
}

static void oracle_block(const int src[16][3], int is_signed, oracle_cand *best)
{
    memset(best, 0, sizeof *best);
    best->err = UINT64_MAX;
    for (int mi = 0; mi < 14; mi++) {
        const bc6h_mode *m = &bc6h_modes[mi];
        const int two = m->regions == 2;
        oracle_cand mb;
        mb.valid = 0;
        mb.err = UINT64_MAX;
        for (int p = 0; p < (two ? 32 : 1); p++) {
            oracle_cand c;
            c.mode = mi;
            c.partition = p;
            for (int s = 0; s < m->regions; s++) {   /* the two texels of the region farthest apart */
                int bi = -1, bj = -1;
                int64_t bd = -1;
                for (int i = 0; i < 16; i++)
                    for (int j = i; j < 16; j++) {
                        if ((two ? bc6h_part[p][i] : 0) != s || (two ? bc6h_part[p][j] : 0) != s) continue;
                        int64_t d = 0;
                        for (int k = 0; k < 3; k++) d += (int64_t)(src[i][k] - src[j][k]) * (src[i][k] - src[j][k]);
                        if (d > bd) { bd = d; bi = i; bj = j; }
                    }
                for (int k = 0; k < 3; k++) {
                    c.q[2 * s][k] = quantize_nearest(target_of(src[bi][k], is_signed), m->prec, is_signed);
                    c.q[2 * s + 1][k] = quantize_nearest(target_of(src[bj][k], is_signed), m->prec, is_signed);
                }
            }
            if (!two) memset(c.q[2], 0, sizeof c.q[2] * 2);
            oracle_eval(src, is_signed, &c);
            oracle_cand cur = c;
            for (int round = 0; round < 2; round++) {
                oracle_cand n = cur;
                for (int s = 0; s < m->regions; s++) {
                    double a[3], b[3];
                    if (!oracle_lsq(src, is_signed, &cur, s, a, b)) continue;
                    for (int k = 0; k < 3; k++) {
                        n.q[2 * s][k] = quantize_nearest(a[k], m->prec, is_signed);
                        n.q[2 * s + 1][k] = quantize_nearest(b[k], m->prec, is_signed);
                    }
                }
                oracle_eval(src, is_signed, &n);
                if (better(&n, &c)) c = n;
                cur = n;
            }
            if (better(&c, &mb)) mb = c;
        }
        if (!mb.valid) continue;
        /* +-1 nudges of each quantised endpoint component, while one helps */
        const int lo = q_lo(m->prec, is_signed), hi = q_hi(m->prec, is_signed);
        for (int improved = 1; improved;) {
            improved = 0;
            for (int e = 0; e < 2 * m->regions; e++)
                for (int k = 0; k < 3; k++)
                    for (int step = -1; step <= 1; step += 2) {
                        oracle_cand n = mb;
                        n.q[e][k] += step;
                        if (n.q[e][k] < lo || n.q[e][k] > hi) continue;
                        oracle_eval(src, is_signed, &n);
                        if (better(&n, &mb)) { mb = n; improved = 1; }
                    }
        }
        if (better(&mb, best)) *best = mb;
    }
}

typedef struct { uint8_t *b; int pos; } bc6h_writer;
static void bc6h_write(bc6h_writer *w, int v, int n)
{
    for (int i = 0; i < n; i++, w->pos++) w->b[w->pos >> 3] |= (uint8_t)(((v >> i) & 1) << (w->pos & 7));
}

static void oracle_pack(const oracle_cand *c, uint8_t blk[16])
{
    const bc6h_mode *m = &bc6h_modes[c->mode];
    int raw[12];
    for (int k = 0; k < 3; k++) {
        raw[k] = c->q[0][k] & ((1 << m->prec) - 1);
        for (int e = 1; e < 4; e++)
            raw[3 * e + k] = m->transformed ? (c->q[e][k] - c->q[0][k]) & ((1 << m->delta[k]) - 1) : c->q[e][k] & ((1 << m->prec) - 1);
    }
    memset(blk, 0, 16);
    bc6h_writer w = {blk, 0};
    bc6h_write(&w, m->mode_value, m->mode_bits);
    for (const bc6h_field *f = m->f; f->comp >= 0; f++) {
        const int step = f->a >= f->b ? 1 : -1;
        for (int k = f->b;; k += step) {
            bc6h_write(&w, (raw[f->comp] >> k) & 1, 1);
            if (k == f->a) break;
        }
    }
    const int two = m->regions == 2, ib = two ? 3 : 4;
    if (two) bc6h_write(&w, c->partition, 5);
    for (int t = 0; t < 16; t++) {
        const int anchor = t == 0 || (two && bc6h_part[c->partition][t] == 1 && t == bc6h_anchor[c->partition]);
        bc6h_write(&w, c->idx[t], anchor ? ib - 1 : ib);
    }
}

/* RGBA16F (4*w halves per row, A ignored) -> blocks row-major over (w/4) x (h/4); errs (may be NULL): per block the error
 * of the block chosen */
void bc6h_oracle_encode(const uint16_t *rgba, int w, int h, int is_signed, uint8_t *blocks, uint64_t *errs)
{
    for (int by = 0; by < h / 4; by++)
        for (int bx = 0; bx < w / 4; bx++) {
            int src[16][3];
            for (int t = 0; t < 16; t++)
                for (int k = 0; k < 3; k++) src[t][k] = src_value(rgba[4 * ((size_t)(4 * by + t / 4) * w + 4 * bx + t % 4) + k], is_signed);
            oracle_cand c;
            oracle_block(src, is_signed, &c);
            const size_t b = (size_t)by * (w / 4) + bx;
            oracle_pack(&c, blocks + 16 * b);
            if (errs) errs[b] = c.err;
        }
}
