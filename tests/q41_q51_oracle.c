/*
 * q41_q51_oracle.c — TEST INFRASTRUCTURE ONLY (same rules as oracle/ggml_oracle.c: only tests/ may load it).
 *
 * The plain-C restatement of the reference's Q4_1 / Q5_1 weights and their Q8_1 activation (AVX2 build), on top of the
 * unchanged oracle: this one translation unit includes oracle/ggml_oracle.c and oracle/llama_oracle.c, renames the
 * former's orc_mul_mat to orc_mul_mat_base and defines an orc_mul_mat that adds types 3 and 7 (the whole-model oracle in
 * llama_oracle.c calls it for every matrix).  Compiled like liboracle.so (-ffp-contract=off): every fused multiply-add
 * below is an explicit fmaf() placed where the reference binary has one.  Line numbers cite models/ggml/ggml.c.
 *
 * Settled against the compiled reference (tests/test_q41_q51.py, tests/golden/kat_q8_1.npz): gcc -O3 -mfma contracts
 * `summs += m * s` in both dots into a fused multiply-add; the unfused chain gives other bits on the known-answer vectors.
 * `x*d + m` in the dequantizers is written fused here, but there the two forms cannot differ: q*d (q <= 31, d an fp16
 * value) needs at most 16 significant bits and is exact in fp32, so rounding it first changes nothing.  orc_q1_set_variant
 * selects the forms the reference does NOT use, for the tests that show which of them the vectors tell apart.
 */
#define orc_mul_mat orc_mul_mat_base
#include "../oracle/ggml_oracle.c"
#undef orc_mul_mat

#define QK4_1 32
#define QK8_1 32

#pragma pack(push, 1)
typedef struct { uint16_t d, m; uint8_t qs[QK4_1 / 2]; } blk_q4_1;                  /* ggml.c:896-900 */
typedef struct { uint16_t d, m; uint8_t qh[4]; uint8_t qs[QK4_1 / 2]; } blk_q5_1;   /* ggml.c:912-917 */
typedef struct { float d, s; int8_t qs[QK8_1]; } blk_q8_1;                          /* ggml.c:928-932 */
#pragma pack(pop)

/* Rejected forms, for the discriminating tests only (0 = the reference's arithmetic). */
enum {
    Q1_SUMMS_UNFUSED = 1,   /* summs = summs + m*s, the product rounded first            */
    Q1_DEQ_UNFUSED = 2,     /* x*d + m, the product rounded first                        */
    Q1_DY_FP16 = 4,         /* Q8_1 d rounded through fp16 as Q8_0's is                  */
    Q1_ROUNDF = 8,          /* q = roundf(x*id) (ties away from zero) instead of ties-to-even */
};
static int g_variant;
void orc_q1_set_variant(int v) { g_variant = v; }

int orc_q1_sizeof_block(int type) {
    switch (type) {
        case 3: return sizeof(blk_q4_1);
        case 7: return sizeof(blk_q5_1);
        case 9: return sizeof(blk_q8_1);
    }
    return orc_sizeof_block(type);
}

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
        if (g_variant & Q1_DY_FP16) d = orc_fp16_to_fp32(orc_fp32_to_fp16(d));
        const float id = (amax != 0.0f) ? 127.f / amax : 0.0f;
        int sum = 0;
        for (int j = 0; j < QK8_1; ++j) {
            const float v = x[i * QK8_1 + j] * id;
            const int q = (int)((g_variant & Q1_ROUNDF) ? roundf(v) : nearbyintf(v));
            y[i].qs[j] = (int8_t)q;
            sum += q;
        }
        y[i].d = d;
        y[i].s = d * (float)sum;
    }
}

static inline float summs_step(float summs, float m, float s) {
    return (g_variant & Q1_SUMMS_UNFUSED) ? summs + m * s : fmaf(m, s, summs);
}
static inline int dot4_u8s8i(const uint8_t *a, const int8_t *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2] + a[3] * b[3]; }

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
        for (int l = 0; l < 8; l++) acc[l] = fmaf(d, (float)dot4_u8s8i(bx + 4 * l, y[i].qs + 4 * l), acc[l]);
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
        for (int l = 0; l < 8; l++) acc[l] = fmaf(d, (float)dot4_u8s8i(bx + 4 * l, y[i].qs + 4 * l), acc[l]);
    }
    return hsum8(acc) + summs;
}

static inline float deq(int q, float d, float m) { return (g_variant & Q1_DEQ_UNFUSED) ? (float)q * d + m : fmaf((float)q, d, m); }

/* ggml.c:1538-1557 dequantize_row_q4_1: x*d + m */
void orc_dequantize_row_q4_1(const void *vx, float *y, int k) {
    const blk_q4_1 *x = (const blk_q4_1 *)vx;
    for (int i = 0; i < k / QK4_1; i++) {
        const float d = orc_fp16_to_fp32(x[i].d), m = orc_fp16_to_fp32(x[i].m);
        for (int j = 0; j < QK4_1 / 2; ++j) {
            y[i * QK4_1 + j] = deq(x[i].qs[j] & 0x0F, d, m);
            y[i * QK4_1 + j + QK4_1 / 2] = deq(x[i].qs[j] >> 4, d, m);
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
            y[i * QK4_1 + j] = deq((x[i].qs[j] & 0x0F) | (int)(((qh >> j) & 1u) << 4), d, m);
            y[i * QK4_1 + j + QK4_1 / 2] = deq((x[i].qs[j] >> 4) | (int)(((qh >> (j + 16)) & 1u) << 4), d, m);
        }
    }
}

/* ggml.c:11031-11245 with the type_traits of ggml.c:1687-1697, 1709-1719: Q4_1 / Q5_1 rows are dotted with the Q8_1 image of
 * each activation row; every other type goes to the oracle's own orc_mul_mat. */
int orc_mul_mat(int type, const void *w, const float *x, float *dst, int K, int M, int N) {
    if (type != 3 && type != 7) return orc_mul_mat_base(type, w, x, dst, K, M, N);
    if (K % QK8_1) return -1;
    const size_t wrow = (size_t)(K / QK8_1) * orc_q1_sizeof_block(type);
    blk_q8_1 *act = (blk_q8_1 *)malloc((size_t)(K / QK8_1) * sizeof(blk_q8_1));
    for (int n = 0; n < N; n++) {
        orc_quantize_row_q8_1(x + (size_t)n * K, act, K);
        for (int m = 0; m < M; m++) {
            const void *wr = (const char *)w + (size_t)m * wrow;
            dst[(size_t)n * M + m] = type == 3 ? orc_vec_dot_q4_1_q8_1(K, wr, act) : orc_vec_dot_q5_1_q8_1(K, wr, act);
        }
    }
    free(act);
    return 0;
}

#include "../oracle/llama_oracle.c"
