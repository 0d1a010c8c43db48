/*
 * tests/bc7_oracle_encode.c -- TEST INFRASTRUCTURE ONLY (never linked into libhap_b200.so).
 *
 * The quality oracle of the library's BC7 encoder (hap_b200/csrc/bc7_encode.cuh), written apart from it: RGBA8 -> BPTC /
 * BC7 RGBA UNORM blocks by an exhaustive sequential search.  It includes the decoder oracle (tests/bc7_oracle.c) whole and
 * packs and scores blocks through that oracle's mode descriptors, partition and anchor tables, weight tables and bc7_interp.
 *   * every mode; every partition (16 for mode 0, 64 for modes 1, 2, 3 and 7); every rotation and index selection;
 *   * per subset: endpoints from the principal axis (double precision), then twice least squares in double precision on
 *     the indices obtained, each under every p-bit choice of the mode; each subset keeps its best;
 *   * the best block of each mode gets +-1 nudges of its endpoint codes until none helps.
 * The error is the sum over R, G, B and A of squared 8-bit differences.  Rules as the kernel's: a block of one colour takes
 * mode 5 at colour index 1 (an endpoint pair found by enumeration here) and decodes exactly; in a block whose texels all have
 * A = 255, modes 4-7 hold the channel that decodes to A at its top code (p-bits 1 in modes 6 and 7).  The reported error is
 * that of bc7_block_texels' decoding of the packed block.
 * Layouts: RGBA8 row-major, stride = 4*w; blocks row-major over (w/4) x (h/4); w, h multiples of 4.
 */
#include "bc7_oracle.c"

#include <math.h>

typedef struct {
    int mode, part, rot, isb;
    int code[6][4];   /* endpoint codes (the mode's bits, p-bit apart) */
    int p[6];         /* p-bit of each endpoint */
    int i1[16], i2[16];
    long err;
} o7_block;

static int o7_expand(int code, int p, int bits, int has_p)
{
    if (bits == 0) return 255;
    int v = has_p ? (code << 1) | p : code, n = bits + has_p;
    v <<= 8 - n;
    return v | (v >> n);
}

/* the code (with p-bit p) whose expansion is nearest v */
static int o7_quant(double v, int bits, int has_p, int p)
{
    int top = (1 << bits) - 1, best = 0;
    double bd = 1e30;
    int guess = (int)floor(v / 255.0 * top + 0.5);
    for (int c = guess - 2; c <= guess + 2; c++) {
        int q = c < 0 ? 0 : c > top ? top : c;
        double d = fabs(o7_expand(q, p, bits, has_p) - v);
        if (d < bd) { bd = d; best = q; }
    }
    return best;
}

static int o7_subset(int mode, int part, int t)
{
    int ns = bc7_modes[mode].ns;
    return ns == 2 ? bc7_part2[part][t] : ns == 3 ? bc7_part3[part][t] : 0;
}

/* the error of subset s of block b on source x (rotated) with every texel at its best index; writes those indices */
static long o7_eval_subset(o7_block *b, int s, const int x[16][4])
{
    const bc7_mode_desc *m = &bc7_modes[b->mode];
    const int has_p = m->epb || m->spb;
    int e0[4], e1[4];
    for (int c = 0; c < 4; c++) {
        int bits = c < 3 ? m->cb : m->ab;
        e0[c] = o7_expand(b->code[2 * s][c], b->p[2 * s], bits, has_p);
        e1[c] = o7_expand(b->code[2 * s + 1][c], b->p[2 * s + 1], bits, has_p);
    }
    long err = 0;
    for (int t = 0; t < 16; t++) {
        if (o7_subset(b->mode, b->part, t) != s) continue;
        if (m->ib2) {
            int cbits = b->isb ? m->ib2 : m->ib, abits = b->isb ? m->ib : m->ib2;
            long bc = -1, ba = -1;
            int ci = 0, ai = 0;
            for (int i = 0; i < (1 << cbits); i++) {
                long d = 0;
                for (int c = 0; c < 3; c++) {
                    int v = bc7_interp(e0[c], e1[c], bc7_weight_of(cbits, i)) - x[t][c];
                    d += (long)v * v;
                }
                if (bc < 0 || d < bc) { bc = d; ci = i; }
            }
            for (int i = 0; i < (1 << abits); i++) {
                int v = bc7_interp(e0[3], e1[3], bc7_weight_of(abits, i)) - x[t][3];
                if (ba < 0 || (long)v * v < ba) { ba = (long)v * v; ai = i; }
            }
            b->i1[t] = b->isb ? ai : ci;
            b->i2[t] = b->isb ? ci : ai;
            err += bc + ba;
        } else {
            long be = -1;
            int bi = 0;
            for (int i = 0; i < (1 << m->ib); i++) {
                long d = 0;
                for (int c = 0; c < 4; c++) {
                    int v = bc7_interp(e0[c], e1[c], bc7_weight_of(m->ib, i)) - x[t][c];
                    d += (long)v * v;
                }
                if (be < 0 || d < be) { be = d; bi = i; }
            }
            b->i1[t] = bi;
            b->i2[t] = 0;
            err += be;
        }
    }
    return err;
}

static long o7_eval(o7_block *b, const int x[16][4])
{
    long e = 0;
    for (int s = 0; s < bc7_modes[b->mode].ns; s++) e += o7_eval_subset(b, s, x);
    return e;
}

/* channels [c0, c1) of subset s: endpoints along the principal axis through the mean, at the extreme projections */
static void o7_axis_fit(const int x[16][4], const int in[16], int c0, int c1, double lo[4], double hi[4])
{
    double mean[4] = {0, 0, 0, 0}, cov[4][4] = {{0}}, n = 0;
    for (int t = 0; t < 16; t++)
        if (in[t]) { n++; for (int c = c0; c < c1; c++) mean[c] += x[t][c]; }
    if (n == 0) return;
    for (int c = c0; c < c1; c++) mean[c] /= n;
    for (int t = 0; t < 16; t++)
        if (in[t])
            for (int i = c0; i < c1; i++)
                for (int j = c0; j < c1; j++) cov[i][j] += (x[t][i] - mean[i]) * (x[t][j] - mean[j]);
    double v[4] = {1, 1, 1, 1};
    for (int it = 0; it < 16; it++) {
        double w[4] = {0, 0, 0, 0}, mx = 0;
        for (int i = c0; i < c1; i++) {
            for (int j = c0; j < c1; j++) w[i] += cov[i][j] * v[j];
            mx = fmax(mx, fabs(w[i]));
        }
        if (mx == 0) break;
        for (int i = c0; i < c1; i++) v[i] = w[i] / mx;
    }
    double tmin = 1e30, tmax = -1e30, vv = 0;
    for (int c = c0; c < c1; c++) vv += v[c] * v[c];
    for (int t = 0; t < 16; t++) {
        if (!in[t]) continue;
        double d = 0;
        for (int c = c0; c < c1; c++) d += (x[t][c] - mean[c]) * v[c];
        d = vv > 0 ? d / vv : 0;
        if (d < tmin) tmin = d;
        if (d > tmax) tmax = d;
    }
    for (int c = c0; c < c1; c++) {
        lo[c] = fmin(255, fmax(0, mean[c] + tmin * v[c]));
        hi[c] = fmin(255, fmax(0, mean[c] + tmax * v[c]));
    }
}

/* least squares for channels [c0, c1) of the texels in `in` with the weights w[t] held */
static void o7_lsq(const int x[16][4], const int in[16], const int w[16], int c0, int c1, double lo[4], double hi[4])
{
    double aa = 0, ab = 0, bb = 0, ax[4] = {0, 0, 0, 0}, bx[4] = {0, 0, 0, 0};
    for (int t = 0; t < 16; t++) {
        if (!in[t]) continue;
        double b = w[t] / 64.0, a = 1 - b;
        aa += a * a; ab += a * b; bb += b * b;
        for (int c = c0; c < c1; c++) { ax[c] += a * x[t][c]; bx[c] += b * x[t][c]; }
    }
    double det = aa * bb - ab * ab;
    if (fabs(det) < 1e-9) return;
    for (int c = c0; c < c1; c++) {
        lo[c] = fmin(255, fmax(0, (bb * ax[c] - ab * bx[c]) / det));
        hi[c] = fmin(255, fmax(0, (aa * bx[c] - ab * ax[c]) / det));
    }
}

/* the stored channel that decodes to A under rotation r */
static int o7_aslot(int rot) { return rot ? rot - 1 : 3; }

/* endpoints of subset s from lo / hi under p-bits (p0, p1); the opaque rule */
static void o7_set(o7_block *b, int s, const double lo[4], const double hi[4], int p0, int p1, int opaque)
{
    const bc7_mode_desc *m = &bc7_modes[b->mode];
    const int has_p = m->epb || m->spb;
    b->p[2 * s] = p0;
    b->p[2 * s + 1] = p1;
    for (int c = 0; c < 4; c++) {
        int bits = c < 3 ? m->cb : m->ab;
        if (bits == 0) { b->code[2 * s][c] = b->code[2 * s + 1][c] = 0; continue; }
        b->code[2 * s][c] = o7_quant(lo[c], bits, has_p, p0);
        b->code[2 * s + 1][c] = o7_quant(hi[c], bits, has_p, p1);
        if (opaque && b->mode >= 4 && c == o7_aslot(b->rot)) b->code[2 * s][c] = b->code[2 * s + 1][c] = (1 << bits) - 1;
    }
}

/* every p-bit choice of subset s, each with the fit and two least-squares refits; subset s of b gets the best */
static long o7_fit_subset(o7_block *b, int s, const int x[16][4], int opaque)
{
    const bc7_mode_desc *m = &bc7_modes[b->mode];
    int in[16];
    for (int t = 0; t < 16; t++) in[t] = o7_subset(b->mode, b->part, t) == s;
    double lo0[4] = {0, 0, 0, 0}, hi0[4] = {0, 0, 0, 0};
    if (m->ib2) { o7_axis_fit(x, in, 0, 3, lo0, hi0); o7_axis_fit(x, in, 3, 4, lo0, hi0); }
    else o7_axis_fit(x, in, 0, 4, lo0, hi0);
    int choices = m->epb ? 4 : m->spb ? 2 : 1;
    if (opaque && b->mode >= 6) choices = 1;
    long best = -1;
    o7_block keep = *b;
    for (int k = 0; k < choices; k++) {
        int p0 = m->epb ? k & 1 : m->spb ? k : 0, p1 = m->epb ? k >> 1 : p0;
        if (opaque && b->mode >= 6) p0 = p1 = 1;
        double lo[4], hi[4];
        memcpy(lo, lo0, sizeof lo);
        memcpy(hi, hi0, sizeof hi);
        for (int it = 0; it < 3; it++) {
            o7_set(b, s, lo, hi, p0, p1, opaque);
            long e = o7_eval_subset(b, s, x);
            if (best < 0 || e < best) { best = e; keep = *b; }
            int w1[16], w2[16];
            for (int t = 0; t < 16; t++) {
                w1[t] = bc7_weight_of(m->ib, b->i1[t]);
                w2[t] = m->ib2 ? bc7_weight_of(m->ib2, b->i2[t]) : 0;
            }
            if (m->ib2) {
                o7_lsq(x, in, b->isb ? w2 : w1, 0, 3, lo, hi);
                o7_lsq(x, in, b->isb ? w1 : w2, 3, 4, lo, hi);
            } else {
                o7_lsq(x, in, w1, 0, 4, lo, hi);
            }
        }
    }
    /* subset s of the kept block, the rest of b unchanged */
    for (int e = 2 * s; e < 2 * s + 2; e++) { memcpy(b->code[e], keep.code[e], sizeof keep.code[e]); b->p[e] = keep.p[e]; }
    for (int t = 0; t < 16; t++)
        if (in[t]) { b->i1[t] = keep.i1[t]; b->i2[t] = keep.i2[t]; }
    return best;
}

/* +-1 nudges of every endpoint code until none lowers the error */
static void o7_nudge(o7_block *b, const int x[16][4], int opaque)
{
    const bc7_mode_desc *m = &bc7_modes[b->mode];
    for (int again = 1; again;) {
        again = 0;
        for (int e = 0; e < 2 * m->ns; e++)
            for (int c = 0; c < 4; c++) {
                int bits = c < 3 ? m->cb : m->ab;
                if (bits == 0 || (opaque && b->mode >= 4 && c == o7_aslot(b->rot))) continue;
                for (int d = -1; d <= 1; d += 2) {
                    int v = b->code[e][c] + d;
                    if (v < 0 || v >= (1 << bits)) continue;
                    o7_block t = *b;
                    t.code[e][c] = v;
                    t.err = o7_eval(&t, x);
                    if (t.err < b->err) { *b = t; again = 1; }
                }
            }
    }
}

typedef struct { uint8_t b[16]; int pos; } o7_writer;
static void o7_put(o7_writer *w, int v, int n)
{
    for (int i = 0; i < n; i++, w->pos++) w->b[w->pos >> 3] |= (uint8_t)(((v >> i) & 1) << (w->pos & 7));
}

/* the block's 128 bits; anchors whose index has its top bit set swap their subset's endpoints and invert its indices */
static void o7_pack(o7_block b, uint8_t out[16])
{
    const bc7_mode_desc *m = &bc7_modes[b.mode];
    int anchor[3] = {0, 0, 0};
    if (m->ns == 2) anchor[1] = bc7_anchor2[b.part];
    if (m->ns == 3) { anchor[1] = bc7_anchor3a[b.part]; anchor[2] = bc7_anchor3b[b.part]; }
    int lo1 = 0, hi1 = 4, lo2 = 4, hi2 = 4;   /* channels each index set drives */
    if (m->ib2) { lo1 = b.isb ? 3 : 0; hi1 = b.isb ? 4 : 3; lo2 = b.isb ? 0 : 3; hi2 = b.isb ? 3 : 4; }
    for (int s = 0; s < m->ns; s++) {
        if (b.i1[anchor[s]] < (1 << (m->ib - 1))) continue;
        for (int c = lo1; c < hi1; c++) { int v = b.code[2 * s][c]; b.code[2 * s][c] = b.code[2 * s + 1][c]; b.code[2 * s + 1][c] = v; }
        if (!m->ib2) { int v = b.p[2 * s]; b.p[2 * s] = b.p[2 * s + 1]; b.p[2 * s + 1] = v; }
        for (int t = 0; t < 16; t++)
            if (o7_subset(b.mode, b.part, t) == s) b.i1[t] = (1 << m->ib) - 1 - b.i1[t];
    }
    if (m->ib2 && b.i2[0] >= (1 << (m->ib2 - 1))) {
        for (int c = lo2; c < hi2; c++) { int v = b.code[0][c]; b.code[0][c] = b.code[1][c]; b.code[1][c] = v; }
        for (int t = 0; t < 16; t++) b.i2[t] = (1 << m->ib2) - 1 - b.i2[t];
    }
    o7_writer w;
    memset(&w, 0, sizeof w);
    o7_put(&w, 1 << b.mode, b.mode + 1);
    o7_put(&w, b.part, m->pb);
    o7_put(&w, b.rot, m->rb);
    o7_put(&w, b.isb, m->isb);
    for (int c = 0; c < 3; c++)
        for (int e = 0; e < 2 * m->ns; e++) o7_put(&w, b.code[e][c], m->cb);
    for (int e = 0; e < 2 * m->ns; e++) o7_put(&w, b.code[e][3], m->ab);
    if (m->epb)
        for (int e = 0; e < 2 * m->ns; e++) o7_put(&w, b.p[e], 1);
    if (m->spb)
        for (int s = 0; s < m->ns; s++) o7_put(&w, b.p[2 * s], 1);
    for (int t = 0; t < 16; t++) {
        int a = 0;
        for (int s = 0; s < m->ns; s++) a |= anchor[s] == t;
        o7_put(&w, b.i1[t], m->ib - a);
    }
    if (m->ib2)
        for (int t = 0; t < 16; t++) o7_put(&w, b.i2[t], m->ib2 - (t == 0));
    memcpy(out, w.b, 16);
}

/* one block: src[t] RGBA of texel t -> 16 bytes; returns the error of the oracle decoder's decoding of them */
static long o7_encode_block(const uint8_t src[16][4], uint8_t out[16])
{
    int flat = 1, opaque = 1;
    for (int t = 0; t < 16; t++) {
        flat &= !memcmp(src[t], src[0], 4);
        opaque &= src[t][3] == 255;
    }
    o7_block best;
    memset(&best, 0, sizeof best);
    best.err = -1;
    if (flat) {
        best.mode = 5;
        for (int c = 0; c < 3; c++) {
            int found = 0;
            for (int a = 0; a < 128 && !found; a++)
                for (int b = 0; b < 128 && !found; b++)
                    if (bc7_interp(o7_expand(a, 0, 7, 0), o7_expand(b, 0, 7, 0), bc7_w2[1]) == src[0][c]) {
                        best.code[0][c] = a;
                        best.code[1][c] = b;
                        found = 1;
                    }
        }
        best.code[0][3] = best.code[1][3] = src[0][3];
        for (int t = 0; t < 16; t++) best.i1[t] = 1;
    } else {
        for (int mode = 0; mode < 8; mode++) {
            const bc7_mode_desc *m = &bc7_modes[mode];
            o7_block mb;
            memset(&mb, 0, sizeof mb);
            mb.err = -1;
            int x[16][4];
            for (int part = 0; part < (1 << m->pb); part++)
                for (int rot = 0; rot < (1 << m->rb); rot++)
                    for (int isb = 0; isb < (1 << m->isb); isb++) {
                        for (int t = 0; t < 16; t++) {
                            for (int c = 0; c < 4; c++) x[t][c] = src[t][c];
                            if (rot) { int v = x[t][3]; x[t][3] = x[t][rot - 1]; x[t][rot - 1] = v; }
                        }
                        o7_block b;
                        memset(&b, 0, sizeof b);
                        b.mode = mode; b.part = part; b.rot = rot; b.isb = isb;
                        long e = 0;
                        for (int s = 0; s < m->ns; s++) e += o7_fit_subset(&b, s, x, opaque);
                        b.err = e;
                        if (mb.err < 0 || e < mb.err) mb = b;
                    }
            for (int t = 0; t < 16; t++) {
                for (int c = 0; c < 4; c++) x[t][c] = src[t][c];
                if (mb.rot) { int v = x[t][3]; x[t][3] = x[t][mb.rot - 1]; x[t][mb.rot - 1] = v; }
            }
            o7_nudge(&mb, x, opaque);
            if (best.err < 0 || mb.err < best.err) best = mb;
        }
    }
    o7_pack(best, out);
    uint8_t dec[16][4];
    bc7_block_texels(out, dec);
    long err = 0;
    for (int t = 0; t < 16; t++)
        for (int c = 0; c < 4; c++) err += (long)(dec[t][c] - src[t][c]) * (dec[t][c] - src[t][c]);
    return err;
}

void bc7_oracle_encode(const uint8_t *rgba, int w, int h, uint8_t *blocks, uint64_t *errs)
{
    for (int by = 0; by < h / 4; by++)
        for (int bx = 0; bx < w / 4; bx++) {
            uint8_t src[16][4];
            for (int t = 0; t < 16; t++) memcpy(src[t], rgba + 4 * ((size_t)(4 * by + t / 4) * w + 4 * bx + t % 4), 4);
            const size_t b = (size_t)by * (w / 4) + bx;
            errs[b] = (uint64_t)o7_encode_block(src, blocks + 16 * b);
        }
}
