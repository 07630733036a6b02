/*
 * q3k_oracle.c — TEST INFRASTRUCTURE ONLY (same rules as ggml_oracle.c): the plain-C restatement of the reference's Q3_K
 * weights (AVX2 build, QK_K = 256).  Compiled like ggml_oracle.c (-ffp-contract=off): the one fused multiply-add per block
 * and AVX lane is an explicit fmaf().  Line numbers cite models/ggml/k_quants.c and k_quants.h.
 */
#include <math.h>
#include <string.h>

#include "ggml_oracle.h"

#pragma pack(push, 1)
typedef struct { uint8_t hmask[QK_K / 8]; uint8_t qs[QK_K / 4]; uint8_t scales[12]; uint16_t d; } blk_q3_K;   /* k_quants.h:55-61 */
#pragma pack(pop)
_Static_assert(sizeof(blk_q3_K) == 110, "orc_sizeof_block(11)");

/* The 16 six-bit scales of a Q3_K block, minus 32 (k_quants.c:593-598 / 1968-1974): with the 12 bytes read as words a0 a1
 * a2, sub-blocks 0..3 take the low nibbles of a0 and bits 0-1 of a2's bytes, 4..7 the low nibbles of a1 and bits 2-3, 8..11
 * the high nibbles of a0 and bits 4-5, 12..15 the high nibbles of a1 and bits 6-7. */
static void q3k_scales(const uint8_t *s, int sc[16]) {
    for (int b = 0; b < 4; b++) {
        sc[b] = ((s[b] & 0xF) | (((s[8 + b] >> 0) & 3) << 4)) - 32;
        sc[4 + b] = ((s[4 + b] & 0xF) | (((s[8 + b] >> 2) & 3) << 4)) - 32;
        sc[8 + b] = ((s[b] >> 4) | (((s[8 + b] >> 4) & 3) << 4)) - 32;
        sc[12 + b] = ((s[4 + b] >> 4) | (((s[8 + b] >> 6) & 3) << 4)) - 32;
    }
}

/* weight e of a block: the 2 low bits from qs[32*(e/128) + e%32] at bit 2*((e%128)/32), minus 4 unless hmask[e%32] has bit e/32 */
static inline int q3k_weight(const blk_q3_K *x, int e) {
    const int g = e >> 5, l = e & 31;
    const int lo = (x->qs[32 * (g >> 2) + l] >> (2 * (g & 3))) & 3;
    return lo - ((x->hmask[l] >> g) & 1 ? 0 : 4);
}

/* k_quants.c:575-623 dequantize_row_q3_K: dl = d * (sc - 32) rounded to float, then dl * q */
void orc_dequantize_row_q3_K(const void *vx, float *y, int k) {
    const blk_q3_K *x = (const blk_q3_K *)vx;
    for (int i = 0; i < k / QK_K; i++) {
        const float d = orc_fp16_to_fp32(x[i].d);
        int sc[16];
        q3k_scales(x[i].scales, sc);
        for (int e = 0; e < QK_K; e++) {
            const int is = 8 * (e >> 7) + 2 * ((e & 127) >> 5) + ((e & 31) >> 4);
            const float dl = d * (float)sc[is];
            y[i * QK_K + e] = dl * (float)q3k_weight(&x[i], e);
        }
    }
}

/* orc_q3k_set_variant(1) selects a form the reference does NOT use: every sub-block's scale times its integer sum taken in
 * float and added to the lane in block order. */
int orc_q3k_variant;   /* orc_q3k_set_variant (variants.c) */

/* k_quants.c:1950-2052 (AVX2 ggml_vec_dot_q3_K_q8_K): int32 lane l holds, for every 32-weight group g, the scale of the
 * 16-weight half the lane lies in (sub-block 2g + l/4) times the sum of weights 4l..4l+3 of the group with their activations;
 * one fma(y.d * d, (float)lane, acc[l]) per block, blocks in order, then hsum_float_8.  The integer part is exact in any
 * order (|q - 4| <= 4, the maddubs pairs stay within +-1024, no saturation); only the fp32 chain has an order. */
float orc_vec_dot_q3_K_q8_K(int n, const void *vx, const void *vy) {
    const blk_q3_K *x = (const blk_q3_K *)vx; const blk_q8_K *y = (const blk_q8_K *)vy;
    const int nb = n / QK_K;
    float acc[8] = {0};
    for (int i = 0; i < nb; ++i) {
        const float d = y[i].d * orc_fp16_to_fp32(x[i].d);
        int sc[16];
        q3k_scales(x[i].scales, sc);
        int32_t sumi[8] = {0};
        for (int g = 0; g < 8; g++)
            for (int l = 0; l < 8; l++) {
                int s = 0;
                for (int t = 0; t < 4; t++) s += q3k_weight(&x[i], 32 * g + 4 * l + t) * y[i].qs[32 * g + 4 * l + t];
                if (orc_q3k_variant == 1) acc[l] = acc[l] + d * ((float)sc[2 * g + (l >> 2)] * (float)s);
                sumi[l] += sc[2 * g + (l >> 2)] * s;
            }
        if (orc_q3k_variant != 1)
            for (int l = 0; l < 8; l++) acc[l] = fmaf(d, (float)sumi[l], acc[l]);
    }
    return hsum8(acc);
}
