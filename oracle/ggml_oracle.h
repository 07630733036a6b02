/*
 * ggml_oracle.h — TEST INFRASTRUCTURE ONLY (see ggml_oracle.c): the block layouts and dot-product helpers that ggml_oracle.c,
 * q3k_oracle.c and q41_q51_oracle.c share, and the functions each file calls in another.
 */
#ifndef GGML_ORACLE_H
#define GGML_ORACLE_H
#include <stddef.h>
#include <stdint.h>

#define QK_K 256
#define QK4_0 32
#define QK8_0 32

/* ------------------------------------------------------------- blocks ---- */
#pragma pack(push, 1)
typedef struct { uint16_t d; uint8_t qs[QK4_0 / 2]; } blk_q4_0;                                   /* ggml.c:888-893  */
typedef struct { uint16_t d; uint8_t qh[4]; uint8_t qs[QK4_0 / 2]; } blk_q5_0;                    /* ggml.c:902-908  */
typedef struct { uint16_t d; int8_t qs[QK8_0]; } blk_q8_0;                                        /* ggml.c:920-925  */
typedef struct { uint16_t d, dmin; uint8_t scales[12]; uint8_t qs[QK_K / 2]; } blk_q4_K;          /* k_quants.h:76-82  */
typedef struct { uint16_t d, dmin; uint8_t scales[12]; uint8_t qh[QK_K / 8]; uint8_t qs[QK_K / 2]; } blk_q5_K; /* k_quants.h:98-104 */
typedef struct { uint8_t ql[QK_K / 2]; uint8_t qh[QK_K / 4]; int8_t scales[QK_K / 16]; uint16_t d; } blk_q6_K; /* k_quants.h:112-117 */
typedef struct { float d; int8_t qs[QK_K]; int16_t bsums[QK_K / 16]; } blk_q8_K;                  /* k_quants.h:121-125 */
#pragma pack(pop)

/* -------------------------------------------------------- dot products ---- */
static inline float hsum8(const float a[8]) {
    float r0 = a[4] + a[0], r1 = a[5] + a[1], r2 = a[6] + a[2], r3 = a[7] + a[3];
    r0 = r0 + r2; r1 = r1 + r3;
    return r0 + r1;
}
static inline int dot4_u8s8(const uint8_t *a, const int8_t *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2] + a[3] * b[3]; }
static inline int dot4_s8s8(const int8_t *a, const int8_t *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2] + a[3] * b[3]; }

float orc_fp16_to_fp32(uint16_t h);
uint16_t orc_fp32_to_fp16(float f);
void orc_quantize_row_q8_K(const float *x, void *vy, int k);

/* Q4_1 / Q5_1 / Q8_1 (q41_q51_oracle.c) and Q3_K (q3k_oracle.c), which orc_mul_mat and the whole-model oracle's get_rows call
 * for those types.  Declared weak: ggml_oracle.c and llama_oracle.c also build, without those files, into an oracle of the
 * other types, and a translation unit that includes them may define these functions itself. */
#define ORC_WEAK __attribute__((weak))
ORC_WEAK void orc_quantize_row_q8_1(const float *x, void *vy, int k);
ORC_WEAK float orc_vec_dot_q4_1_q8_1(int n, const void *vx, const void *vy);
ORC_WEAK float orc_vec_dot_q5_1_q8_1(int n, const void *vx, const void *vy);
ORC_WEAK float orc_vec_dot_q3_K_q8_K(int n, const void *vx, const void *vy);
ORC_WEAK void orc_dequantize_row_q4_1(const void *vx, float *y, int k);
ORC_WEAK void orc_dequantize_row_q5_1(const void *vx, float *y, int k);
ORC_WEAK void orc_dequantize_row_q3_K(const void *vx, float *y, int k);
#endif
