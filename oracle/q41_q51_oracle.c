/*
 * q41_q51_oracle.c — TEST INFRASTRUCTURE ONLY (same rules as ggml_oracle.c): the plain-C restatement of the reference's Q4_1 /
 * Q5_1 weights and their Q8_1 activation (AVX2 build).  Compiled like ggml_oracle.c (-ffp-contract=off): every fused
 * multiply-add below is an explicit fmaf() placed where the reference binary has one.  Line numbers cite models/ggml/ggml.c.
 */
#include <math.h>
#include <string.h>

#include "ggml_oracle.h"

#define QK4_1 32
#define QK8_1 32

#pragma pack(push, 1)
typedef struct { uint16_t d, m; uint8_t qs[QK4_1 / 2]; } blk_q4_1;                  /* ggml.c:896-900 */
typedef struct { uint16_t d, m; uint8_t qh[4]; uint8_t qs[QK4_1 / 2]; } blk_q5_1;   /* ggml.c:912-917 */
typedef struct { float d, s; int8_t qs[QK8_1]; } blk_q8_1;                          /* ggml.c:928-932 */
#pragma pack(pop)
_Static_assert(sizeof(blk_q4_1) == 20 && sizeof(blk_q5_1) == 24 && sizeof(blk_q8_1) == 40, "orc_sizeof_block(3, 7, 9)");

/* Q4_1 / Q5_1 / Q8_1 forms the reference does NOT use (orc_q1_set_variant bits; 0 = the reference's arithmetic).  Settled
 * against the compiled reference (tests/golden/kat_q8_1.npz): gcc -O3 -mfma contracts `summs += m * s` in both dots into a
 * fused multiply-add; the unfused chain gives other bits on the known-answer vectors.  `x*d + m` in the dequantizers is
 * written fused, but there the two forms cannot differ: q*d (q <= 31, d an fp16 value) needs at most 16 significant bits and
 * is exact in fp32, so rounding it first changes nothing. */
enum {
    Q1_SUMMS_UNFUSED = 1,   /* summs = summs + m*s, the product rounded first            */
    Q1_DEQ_UNFUSED = 2,     /* x*d + m, the product rounded first                        */
    Q1_DY_FP16 = 4,         /* Q8_1 d rounded through fp16 as Q8_0's is                  */
    Q1_ROUNDF = 8,          /* q = roundf(x*id) (ties away from zero) instead of ties-to-even */
};
int orc_q1_variant;   /* orc_q1_set_variant (variants.c) */

/* ggml.c:1420-1481, AVX2 quantize_row_q8_1: amax per 32, d = amax/127 kept as a float (not rounded to fp16 as Q8_0's),
 * id = 127/amax, q = round-half-even(x*id) (_mm256_round_ps NEAREST on the rounded product), s = d * (float)Σq (the
 * integer sum is exact; one float multiply). */
void orc_quantize_row_q8_1(const float *x, void *vy, int k) {
    blk_q8_1 *y = (blk_q8_1 *)vy;
    const int nb = k / QK8_1;
    for (int i = 0; i < nb; i++) {
        float amax = 0.0f;
        for (int j = 0; j < QK8_1; j++) {
            const float a = fabsf(x[i * QK8_1 + j]);
            if (a > amax) amax = a;
        }
        float d = amax / 127.f;
        if (orc_q1_variant & Q1_DY_FP16) d = orc_fp16_to_fp32(orc_fp32_to_fp16(d));
        const float id = (amax != 0.0f) ? 127.f / amax : 0.0f;
        int sum = 0;
        for (int j = 0; j < QK8_1; ++j) {
            const float v = x[i * QK8_1 + j] * id;
            const int q = (int)((orc_q1_variant & Q1_ROUNDF) ? roundf(v) : nearbyintf(v));
            y[i].qs[j] = (int8_t)q;
            sum += q;
        }
        y[i].d = d;
        y[i].s = d * (float)sum;
    }
}

static inline float deq_q1(int q, float d, float m) { return (orc_q1_variant & Q1_DEQ_UNFUSED) ? (float)q * d + m : fmaf((float)q, d, m); }

/* ggml.c:1538-1557 dequantize_row_q4_1: x*d + m */
void orc_dequantize_row_q4_1(const void *vx, float *y, int k) {
    const blk_q4_1 *x = (const blk_q4_1 *)vx;
    for (int i = 0; i < k / QK4_1; i++) {
        const float d = orc_fp16_to_fp32(x[i].d), m = orc_fp16_to_fp32(x[i].m);
        for (int j = 0; j < QK4_1 / 2; ++j) {
            y[i * QK4_1 + j] = deq_q1(x[i].qs[j] & 0x0F, d, m);
            y[i * QK4_1 + j + QK4_1 / 2] = deq_q1(x[i].qs[j] >> 4, d, m);
        }
    }
}

/* ggml.c:1585-1610 dequantize_row_q5_1: the fifth bit of element j is bit j of qh */
void orc_dequantize_row_q5_1(const void *vx, float *y, int k) {
    const blk_q5_1 *x = (const blk_q5_1 *)vx;
    for (int i = 0; i < k / QK4_1; i++) {
        const float d = orc_fp16_to_fp32(x[i].d), m = orc_fp16_to_fp32(x[i].m);
        uint32_t qh; memcpy(&qh, x[i].qh, sizeof(qh));
        for (int j = 0; j < QK4_1 / 2; ++j) {
            y[i * QK4_1 + j] = deq_q1((x[i].qs[j] & 0x0F) | (int)(((qh >> j) & 1u) << 4), d, m);
            y[i * QK4_1 + j + QK4_1 / 2] = deq_q1((x[i].qs[j] >> 4) | (int)(((qh >> (j + 16)) & 1u) << 4), d, m);
        }
    }
}

static inline float summs_step(float summs, float m, float s) {
    return (orc_q1_variant & Q1_SUMMS_UNFUSED) ? summs + m * s : fmaf(m, s, summs);
}

/* ggml.c:2770-2803 (AVX2 ggml_vec_dot_q4_1_q8_1): bytes_from_nibbles_32 (unsigned, no -8) and mul_sum_us8_pairs_float leave the
 * integer sum of elements 4l..4l+3 in lane l; acc = fma(d_w*d_y, lane, acc) per block in block order; the mins term is the
 * scalar chain summs += m_w * s_y in block order; result hsum_float_8(acc) + summs. */
float orc_vec_dot_q4_1_q8_1(int n, const void *vx, const void *vy) {
    const blk_q4_1 *x = (const blk_q4_1 *)vx; const blk_q8_1 *y = (const blk_q8_1 *)vy;
    const int nb = n / QK8_1;
    float acc[8] = {0};
    float summs = 0.f;
    for (int i = 0; i < nb; i++) {
        const float d = orc_fp16_to_fp32(x[i].d) * y[i].d;
        summs = summs_step(summs, orc_fp16_to_fp32(x[i].m), y[i].s);
        uint8_t bx[32];
        for (int j = 0; j < 16; j++) { bx[j] = x[i].qs[j] & 0x0F; bx[j + 16] = x[i].qs[j] >> 4; }
        for (int l = 0; l < 8; l++) acc[l] = fmaf(d, (float)dot4_u8s8(bx + 4 * l, y[i].qs + 4 * l), acc[l]);
    }
    return hsum8(acc) + summs;
}

/* ggml.c:3234-3259 (AVX2 ggml_vec_dot_q5_1_q8_1): the nibbles with bit j of qh ORed in as 0x10 (value 0..31, no -16);
 * acc = fma(lane, d_w*d_y, acc) — the same fused value as Q4_1's operand order. */
float orc_vec_dot_q5_1_q8_1(int n, const void *vx, const void *vy) {
    const blk_q5_1 *x = (const blk_q5_1 *)vx; const blk_q8_1 *y = (const blk_q8_1 *)vy;
    const int nb = n / QK8_1;
    float acc[8] = {0};
    float summs = 0.f;
    for (int i = 0; i < nb; i++) {
        const float d = orc_fp16_to_fp32(x[i].d) * y[i].d;
        summs = summs_step(summs, orc_fp16_to_fp32(x[i].m), y[i].s);
        uint32_t qh; memcpy(&qh, x[i].qh, sizeof(qh));
        uint8_t bx[32];
        for (int j = 0; j < 16; j++) {
            bx[j] = (uint8_t)((x[i].qs[j] & 0x0F) | (((qh >> j) & 1u) << 4));
            bx[j + 16] = (uint8_t)((x[i].qs[j] >> 4) | (((qh >> (j + 16)) & 1u) << 4));
        }
        for (int l = 0; l < 8; l++) acc[l] = fmaf(d, (float)dot4_u8s8(bx + 4 * l, y[i].qs + 4 * l), acc[l]);
    }
    return hsum8(acc) + summs;
}
