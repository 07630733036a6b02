/*
 * head_dims_oracle.c — TEST INFRASTRUCTURE ONLY (same rules as oracle/ggml_oracle.c: only tests/ may load it).
 *
 * The unchanged oracle (oracle/ggml_oracle.c + oracle/llama_oracle.c in one translation unit), with the whole-model
 * oracle's attention head routed through orc_attn_head_hd.  With variant 0 that is orc_attn_head_n itself, the reference's
 * arithmetic.  The other variants change only the K·q dot's tail (elements head_dim & ~31 .. head_dim-1, ggml.c:2415-2418),
 * for the tests that show the stored reference results tell these forms apart:
 *   1  the tail summed in fp32 after the lane reduction, not in double
 *   2  the tail folded into the 4 x 8 lanes (as if the row were zero-padded to a multiple of 32), no scalar part
 * Compiled like liboracle.so (-ffp-contract=off).
 */
#include "../oracle/ggml_oracle.c"

static int g_hd_variant;
void orc_hd_set_variant(int v) { g_hd_variant = v; }

static float kq_dot_variant(int n, const uint16_t *x, const uint16_t *y) {
    float sum[4][8];
    memset(sum, 0, sizeof(sum));
    const int np = n & ~31, nl = g_hd_variant == 2 ? (n + 31) & ~31 : np;
    for (int i = 0; i < nl; i += 32)
        for (int j = 0; j < 4; j++)
            for (int l = 0; l < 8; l++) {
                const int e = i + 8 * j + l;
                if (e < n) sum[j][l] = fmaf(orc_fp16_to_fp32(x[e]), orc_fp16_to_fp32(y[e]), sum[j][l]);
            }
    float t0[4];
    for (int l = 0; l < 8; l++) { sum[0][l] = sum[0][l] + sum[2][l]; sum[1][l] = sum[1][l] + sum[3][l]; }
    for (int l = 0; l < 8; l++) sum[0][l] = sum[0][l] + sum[1][l];
    for (int l = 0; l < 4; l++) t0[l] = sum[0][l] + sum[0][l + 4];
    float res = (t0[0] + t0[1]) + (t0[2] + t0[3]);
    if (g_hd_variant == 1)
        for (int i = np; i < n; ++i) res += orc_fp16_to_fp32(x[i]) * orc_fp16_to_fp32(y[i]);
    return res;
}

/* orc_attn_head_n (oracle/ggml_oracle.c) with the K·q dot of the selected variant; the rest is the same code */
void orc_attn_head_hd(const float *q, const uint16_t *kcache, size_t k_stride, const uint16_t *vcache, size_t v_stride,
                      int head_dim, int T, int n_total, float kq_scale, float *out) {
    if (g_hd_variant == 0) {
        orc_attn_head_n(q, kcache, k_stride, vcache, v_stride, head_dim, T, n_total, kq_scale, out);
        return;
    }
    uint16_t *q16 = (uint16_t *)malloc(sizeof(uint16_t) * head_dim);
    float *s = (float *)malloc(sizeof(float) * n_total);
    uint16_t *p16 = (uint16_t *)calloc((size_t)n_total, sizeof(uint16_t));
    orc_fp32_to_fp16_row(q, q16, head_dim);
    for (int t = 0; t < T; t++) s[t] = kq_dot_variant(head_dim, kcache + (size_t)t * k_stride, q16) * kq_scale;
    orc_soft_max(s, s, T);
    orc_fp32_to_fp16_row(s, p16, T);
    for (int c = 0; c < head_dim; c++) out[c] = orc_vec_dot_f16(n_total, vcache + (size_t)c * v_stride, p16);
    free(q16); free(s); free(p16);
}

#define orc_attn_head_n orc_attn_head_hd
#include "../oracle/llama_oracle.c"
#undef orc_attn_head_n
