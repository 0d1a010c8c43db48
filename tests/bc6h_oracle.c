/*
 * tests/bc6h_oracle.c -- TEST INFRASTRUCTURE ONLY (never linked into libhap_b200.so).
 *
 * The oracle of the library's BC6H decoder (hap_b200/csrc/bc6h_decode.cuh), written apart from it: BPTC / BC6H
 * (RGB UNSIGNED_FLOAT "UF16" and SIGNED_FLOAT "SF16") blocks -> RGBA16F, restated from the format in its plain sequential
 * form.  Each mode's header is a list of fields in the order the block stores them, in the specification's notation:
 * {endpoint component, a, b} is component[a:b], whose first stored bit is bit b; a < b is one of the reversed runs of
 * modes 13 and 14.  The partition table is the specification's 32 two-region partitions as subset lists.
 * Checked in tests/test_bc6h_cpu.py against Pillow's independent "bcn" decoder.  Built by tests/bc6h_util.py.
 * Layouts: RGBA16F (R, G, B, A binary16, A = 1.0) row-major, 4*w values per row; blocks row-major over (w/4) x (h/4).
 */
#include <stddef.h>
#include <stdint.h>
#include <string.h>

static const uint8_t bc6h_part[32][16] = {
    {0, 0, 1, 1, 0, 0, 1, 1, 0, 0, 1, 1, 0, 0, 1, 1}, {0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0, 1},
    {0, 1, 1, 1, 0, 1, 1, 1, 0, 1, 1, 1, 0, 1, 1, 1}, {0, 0, 0, 1, 0, 0, 1, 1, 0, 0, 1, 1, 0, 1, 1, 1},
    {0, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 1, 1}, {0, 0, 1, 1, 0, 1, 1, 1, 0, 1, 1, 1, 1, 1, 1, 1},
    {0, 0, 0, 1, 0, 0, 1, 1, 0, 1, 1, 1, 1, 1, 1, 1}, {0, 0, 0, 0, 0, 0, 0, 1, 0, 0, 1, 1, 0, 1, 1, 1},
    {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 0, 0, 1, 1}, {0, 0, 1, 1, 0, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1},
    {0, 0, 0, 0, 0, 0, 0, 1, 0, 1, 1, 1, 1, 1, 1, 1}, {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 0, 1, 1, 1},
    {0, 0, 0, 1, 0, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1}, {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1},
    {0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1}, {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1},
    {0, 0, 0, 0, 1, 0, 0, 0, 1, 1, 1, 0, 1, 1, 1, 1}, {0, 1, 1, 1, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0, 0},
    {0, 0, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 1, 1, 1, 0}, {0, 1, 1, 1, 0, 0, 1, 1, 0, 0, 0, 1, 0, 0, 0, 0},
    {0, 0, 1, 1, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0, 0}, {0, 0, 0, 0, 1, 0, 0, 0, 1, 1, 0, 0, 1, 1, 1, 0},
    {0, 0, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 1, 1, 0, 0}, {0, 1, 1, 1, 0, 0, 1, 1, 0, 0, 1, 1, 0, 0, 0, 1},
    {0, 0, 1, 1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0, 0}, {0, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0, 1, 1, 0, 0},
    {0, 1, 1, 0, 0, 1, 1, 0, 0, 1, 1, 0, 0, 1, 1, 0}, {0, 0, 1, 1, 0, 1, 1, 0, 0, 1, 1, 0, 1, 1, 0, 0},
    {0, 0, 0, 1, 0, 1, 1, 1, 1, 1, 1, 0, 1, 0, 0, 0}, {0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0},
    {0, 1, 1, 1, 0, 0, 0, 1, 1, 0, 0, 0, 1, 1, 1, 0}, {0, 0, 1, 1, 1, 0, 0, 1, 1, 0, 0, 1, 1, 1, 0, 0},
};
/* the texel of subset 1 whose index is stored with one bit less (texel 0 is that of subset 0) */
static const uint8_t bc6h_anchor[32] = {15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15,
                                        15, 2, 8, 2, 2, 8, 8, 15, 2, 8, 2, 2, 8, 8, 2, 2};

/* endpoint components: w = r0 g0 b0 (0-2), x = r1 g1 b1 (3-5), y = r2 g2 b2 (6-8), z = r3 g3 b3 (9-11) */
enum { R0, G0, B0, R1, G1, B1, R2, G2, B2, R3, G3, B3 };
typedef struct { int8_t comp, a, b; } bc6h_field;   /* comp[a:b]; comp = -1 ends the list */
typedef struct {
    int mode_bits, mode_value, regions, transformed, prec, delta[3];
    bc6h_field f[24];
} bc6h_mode;

#define E {-1, 0, 0}
static const bc6h_mode bc6h_modes[14] = {
    /* 1 */ {2, 0x00, 2, 1, 10, {5, 5, 5}, {{G2, 4, 4}, {B2, 4, 4}, {B3, 4, 4}, {R0, 9, 0}, {G0, 9, 0}, {B0, 9, 0}, {R1, 4, 0},
             {G3, 4, 4}, {G2, 3, 0}, {G1, 4, 0}, {B3, 0, 0}, {G3, 3, 0}, {B1, 4, 0}, {B3, 1, 1}, {B2, 3, 0}, {R2, 4, 0},
             {B3, 2, 2}, {R3, 4, 0}, {B3, 3, 3}, E}},
    /* 2 */ {2, 0x01, 2, 1, 7, {6, 6, 6}, {{G2, 5, 5}, {G3, 4, 4}, {G3, 5, 5}, {R0, 6, 0}, {B3, 0, 0}, {B3, 1, 1}, {B2, 4, 4},
             {G0, 6, 0}, {B2, 5, 5}, {B3, 2, 2}, {G2, 4, 4}, {B0, 6, 0}, {B3, 3, 3}, {B3, 5, 5}, {B3, 4, 4}, {R1, 5, 0},
             {G2, 3, 0}, {G1, 5, 0}, {G3, 3, 0}, {B1, 5, 0}, {B2, 3, 0}, {R2, 5, 0}, {R3, 5, 0}, E}},
    /* 3 */ {5, 0x02, 2, 1, 11, {5, 4, 4}, {{R0, 9, 0}, {G0, 9, 0}, {B0, 9, 0}, {R1, 4, 0}, {R0, 10, 10}, {G2, 3, 0}, {G1, 3, 0},
             {G0, 10, 10}, {B3, 0, 0}, {G3, 3, 0}, {B1, 3, 0}, {B0, 10, 10}, {B3, 1, 1}, {B2, 3, 0}, {R2, 4, 0}, {B3, 2, 2},
             {R3, 4, 0}, {B3, 3, 3}, E}},
    /* 4 */ {5, 0x06, 2, 1, 11, {4, 5, 4}, {{R0, 9, 0}, {G0, 9, 0}, {B0, 9, 0}, {R1, 3, 0}, {R0, 10, 10}, {G3, 4, 4}, {G2, 3, 0},
             {G1, 4, 0}, {G0, 10, 10}, {G3, 3, 0}, {B1, 3, 0}, {B0, 10, 10}, {B3, 1, 1}, {B2, 3, 0}, {R2, 3, 0}, {B3, 0, 0},
             {B3, 2, 2}, {R3, 3, 0}, {G2, 4, 4}, {B3, 3, 3}, E}},
    /* 5 */ {5, 0x0A, 2, 1, 11, {4, 4, 5}, {{R0, 9, 0}, {G0, 9, 0}, {B0, 9, 0}, {R1, 3, 0}, {R0, 10, 10}, {B2, 4, 4}, {G2, 3, 0},
             {G1, 3, 0}, {G0, 10, 10}, {B3, 0, 0}, {G3, 3, 0}, {B1, 4, 0}, {B0, 10, 10}, {B2, 3, 0}, {R2, 3, 0}, {B3, 1, 1},
             {B3, 2, 2}, {R3, 3, 0}, {B3, 4, 4}, {B3, 3, 3}, E}},
    /* 6 */ {5, 0x0E, 2, 1, 9, {5, 5, 5}, {{R0, 8, 0}, {B2, 4, 4}, {G0, 8, 0}, {G2, 4, 4}, {B0, 8, 0}, {B3, 4, 4}, {R1, 4, 0},
             {G3, 4, 4}, {G2, 3, 0}, {G1, 4, 0}, {B3, 0, 0}, {G3, 3, 0}, {B1, 4, 0}, {B3, 1, 1}, {B2, 3, 0}, {R2, 4, 0},
             {B3, 2, 2}, {R3, 4, 0}, {B3, 3, 3}, E}},
    /* 7 */ {5, 0x12, 2, 1, 8, {6, 5, 5}, {{R0, 7, 0}, {G3, 4, 4}, {B2, 4, 4}, {G0, 7, 0}, {B3, 2, 2}, {G2, 4, 4}, {B0, 7, 0},
             {B3, 3, 3}, {B3, 4, 4}, {R1, 5, 0}, {G2, 3, 0}, {G1, 4, 0}, {B3, 0, 0}, {G3, 3, 0}, {B1, 4, 0}, {B3, 1, 1},
             {B2, 3, 0}, {R2, 5, 0}, {R3, 5, 0}, E}},
    /* 8 */ {5, 0x16, 2, 1, 8, {5, 6, 5}, {{R0, 7, 0}, {B3, 0, 0}, {B2, 4, 4}, {G0, 7, 0}, {G2, 5, 5}, {G2, 4, 4}, {B0, 7, 0},
             {G3, 5, 5}, {B3, 4, 4}, {R1, 4, 0}, {G3, 4, 4}, {G2, 3, 0}, {G1, 5, 0}, {G3, 3, 0}, {B1, 4, 0}, {B3, 1, 1},
             {B2, 3, 0}, {R2, 4, 0}, {B3, 2, 2}, {R3, 4, 0}, {B3, 3, 3}, E}},
    /* 9 */ {5, 0x1A, 2, 1, 8, {5, 5, 6}, {{R0, 7, 0}, {B3, 1, 1}, {B2, 4, 4}, {G0, 7, 0}, {B2, 5, 5}, {G2, 4, 4}, {B0, 7, 0},
             {B3, 5, 5}, {B3, 4, 4}, {R1, 4, 0}, {G3, 4, 4}, {G2, 3, 0}, {G1, 4, 0}, {B3, 0, 0}, {G3, 3, 0}, {B1, 5, 0},
             {B2, 3, 0}, {R2, 4, 0}, {B3, 2, 2}, {R3, 4, 0}, {B3, 3, 3}, E}},
    /* 10 */ {5, 0x1E, 2, 0, 6, {6, 6, 6}, {{R0, 5, 0}, {G3, 4, 4}, {B3, 0, 0}, {B3, 1, 1}, {B2, 4, 4}, {G0, 5, 0}, {G2, 5, 5},
              {B2, 5, 5}, {B3, 2, 2}, {G2, 4, 4}, {B0, 5, 0}, {G3, 5, 5}, {B3, 3, 3}, {B3, 5, 5}, {B3, 4, 4}, {R1, 5, 0},
              {G2, 3, 0}, {G1, 5, 0}, {G3, 3, 0}, {B1, 5, 0}, {B2, 3, 0}, {R2, 5, 0}, {R3, 5, 0}, E}},
    /* 11 */ {5, 0x03, 1, 0, 10, {10, 10, 10}, {{R0, 9, 0}, {G0, 9, 0}, {B0, 9, 0}, {R1, 9, 0}, {G1, 9, 0}, {B1, 9, 0}, E}},
    /* 12 */ {5, 0x07, 1, 1, 11, {9, 9, 9}, {{R0, 9, 0}, {G0, 9, 0}, {B0, 9, 0}, {R1, 8, 0}, {R0, 10, 10}, {G1, 8, 0},
              {G0, 10, 10}, {B1, 8, 0}, {B0, 10, 10}, E}},
    /* 13 */ {5, 0x0B, 1, 1, 12, {8, 8, 8}, {{R0, 9, 0}, {G0, 9, 0}, {B0, 9, 0}, {R1, 7, 0}, {R0, 10, 11}, {G1, 7, 0},
              {G0, 10, 11}, {B1, 7, 0}, {B0, 10, 11}, E}},
    /* 14 */ {5, 0x0F, 1, 1, 16, {4, 4, 4}, {{R0, 9, 0}, {G0, 9, 0}, {B0, 9, 0}, {R1, 3, 0}, {R0, 10, 15}, {G1, 3, 0},
              {G0, 10, 15}, {B1, 3, 0}, {B0, 10, 15}, E}},
};
#undef E

static const int bc6h_w3[8] = {0, 9, 18, 27, 37, 46, 55, 64};
static const int bc6h_w4[16] = {0, 4, 9, 13, 17, 21, 26, 30, 34, 38, 43, 47, 51, 55, 60, 64};

typedef struct { const uint8_t *b; int pos; } bc6h_reader;
static int bc6h_read(bc6h_reader *r, int n)
{
    int v = 0;
    for (int i = 0; i < n; i++, r->pos++) v |= ((r->b[r->pos >> 3] >> (r->pos & 7)) & 1) << i;
    return v;
}

static int sign_extend(int v, int bits) { return (v & (1 << (bits - 1))) ? v - (1 << bits) : v; }

/* mode number (0-based index into bc6h_modes) of a block, -1 for the four reserved 5-bit mode values */
static int bc6h_mode_of(const uint8_t *blk)
{
    for (int m = 0; m < 14; m++)
        if ((blk[0] & ((1 << bc6h_modes[m].mode_bits) - 1)) == bc6h_modes[m].mode_value) return m;
    return -1;
}

static int unquantize(int v, int prec, int is_signed)
{
    if (!is_signed) {
        if (prec >= 15) return v;
        if (v == 0) return 0;
        if (v == (1 << prec) - 1) return 0xFFFF;
        return ((v << 16) + 0x8000) >> prec;
    }
    /* -32768 would scale to the bits of -Inf (0xFC00): taken as -32767, so that every output is finite */
    if (prec >= 16) return v < -32767 ? -32767 : v;
    int neg = v < 0, a = neg ? -v : v, q;
    if (a == 0) q = 0;
    else if (a >= (1 << (prec - 1)) - 1) q = 0x7FFF;
    else q = ((a << 15) + 0x4000) >> (prec - 1);
    return neg ? -q : q;
}

/* the interpolated value -> its binary16 bits.  A negative value whose magnitude scales to 0 gives +0 (0x0000). */
static uint16_t finish(int v, int is_signed)
{
    if (!is_signed) return (uint16_t)((v * 31) >> 6);
    if (v < 0) {
        int m = ((-v) * 31) >> 5;
        return (uint16_t)(m ? 0x8000 | m : 0);
    }
    return (uint16_t)((v * 31) >> 5);
}

static void bc6h_block_texels(const uint8_t *blk, int is_signed, int round, uint16_t out[16][4])
{
    const int mi = bc6h_mode_of(blk);
    if (mi < 0) {
        for (int t = 0; t < 16; t++) { out[t][0] = out[t][1] = out[t][2] = 0; out[t][3] = 0x3C00; }
        return;
    }
    const bc6h_mode *m = &bc6h_modes[mi];
    bc6h_reader r = {blk, m->mode_bits};
    int ep[12];
    memset(ep, 0, sizeof ep);
    for (const bc6h_field *f = m->f; f->comp >= 0; f++) {
        const int step = f->a >= f->b ? 1 : -1;
        for (int k = f->b;; k += step) {
            ep[f->comp] |= bc6h_read(&r, 1) << k;
            if (k == f->a) break;
        }
    }
    const int ne = 2 * m->regions, partition = m->regions == 2 ? bc6h_read(&r, 5) : 0;
    /* endpoints: sign extension, the inverse transform */
    for (int c = 0; c < 3; c++) {
        if (is_signed) ep[c] = sign_extend(ep[c], m->prec);
        for (int e = 1; e < ne; e++) {
            int v = ep[3 * e + c];
            if (m->transformed) {
                v = (sign_extend(v, m->delta[c]) + ep[c]) & ((1 << m->prec) - 1);
                if (is_signed) v = sign_extend(v, m->prec);
            } else if (is_signed) {
                v = sign_extend(v, m->prec);
            }
            ep[3 * e + c] = v;
        }
    }
    for (int k = 0; k < 3 * ne; k++) ep[k] = unquantize(ep[k], m->prec, is_signed);
    const int ib = m->regions == 2 ? 3 : 4;
    for (int t = 0; t < 16; t++) {
        const int s = m->regions == 2 ? bc6h_part[partition][t] : 0;
        const int anchor = t == 0 || (s == 1 && t == bc6h_anchor[partition]);
        const int idx = bc6h_read(&r, anchor ? ib - 1 : ib);
        const int w = ib == 3 ? bc6h_w3[idx] : bc6h_w4[idx];
        for (int c = 0; c < 3; c++) {
            const int a = ep[6 * s + c], b = ep[6 * s + 3 + c];
            out[t][c] = finish((a * (64 - w) + b * w + round) >> 6, is_signed);
        }
        out[t][3] = 0x3C00;
    }
}

/* blocks -> RGBA16F.  round: the interpolation's rounding term, 32 as the specification says (0: truncating, as Pillow) */
void bc6h_oracle_decode(const uint8_t *blocks, int w, int h, int is_signed, int round, uint16_t *rgba)
{
    int bw = w / 4, bh = h / 4;
    for (int by = 0; by < bh; by++)
        for (int bx = 0; bx < bw; bx++) {
            uint16_t tex[16][4];
            bc6h_block_texels(blocks + 16 * ((size_t)by * bw + bx), is_signed, round, tex);
            for (int t = 0; t < 16; t++) memcpy(rgba + 4 * ((size_t)(4 * by + t / 4) * w + 4 * bx + t % 4), tex[t], 8);
        }
}

/* What the oracle knows of mode `mode` (0-13), for test writers: its mode bits and value, regions, transformed, precision
 * and delta bits, and per header bit p < 82 the endpoint component (comp[p], -1 for mode and partition bits) and
 * component bit it carries.  Returns the header length in bits (mode + endpoints + partition). */
int bc6h_oracle_layout(int mode, int info[8], int8_t comp[82], int8_t bit[82])
{
    const bc6h_mode *m = &bc6h_modes[mode];
    info[0] = m->mode_bits; info[1] = m->mode_value; info[2] = m->regions; info[3] = m->transformed;
    info[4] = m->prec; info[5] = m->delta[0]; info[6] = m->delta[1]; info[7] = m->delta[2];
    memset(comp, -1, 82);
    memset(bit, 0, 82);
    int p = m->mode_bits;
    for (const bc6h_field *f = m->f; f->comp >= 0; f++) {
        const int step = f->a >= f->b ? 1 : -1;
        for (int k = f->b;; k += step) {
            comp[p] = f->comp;
            bit[p++] = (int8_t)k;
            if (k == f->a) break;
        }
    }
    return p + (m->regions == 2 ? 5 : 0);
}

/* the partition table and anchors the oracle uses: part[32][16], anchor[32] */
void bc6h_oracle_tables(uint8_t *part, uint8_t *anchor)
{
    memcpy(part, bc6h_part, sizeof bc6h_part);
    memcpy(anchor, bc6h_anchor, sizeof bc6h_anchor);
}
