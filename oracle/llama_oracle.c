/*
 * llama_oracle.c — TEST INFRASTRUCTURE ONLY (see ggml_oracle.c header; same rules: only tests/, smoke() and
 * bench.py's cpu_baseline leg may load this).
 *
 * Plain-C, single-threaded restatement of the reference's whole eval for the two GGUF graph shapes:
 *   llm_build_llama   models/ggml/llama.cpp:2162-2491
 *   llm_build_falcon  models/ggml/llama.cpp:2493-2798
 *   driver            llama_eval_internal, models/ggml/llama.cpp:2835-2981 (last token's logits / result_norm row)
 * built from the per-op restatements in ggml_oracle.c (each cites its own reference lines).  Token by token:
 * the reference evaluates a batch of N tokens with exactly the same per-token arithmetic (every src1 row is quantized
 * and dotted independently, ggml.c:11141-11244; attention row n sees positions <= n_past+n, ggml.c:11925-11973),
 * so a sequential restatement produces the same numbers — provided each token's V·P dot is taken over the n_past + N
 * columns of ITS eval call (the f16 dot's SIMD/scalar split depends on that length), which orc_eval does: call it with the
 * same token chunks the reference's BatchEval uses (llm.h:40-54).
 *
 * KV cache layout follows the reference: K [layer][n_ctx][n_embd_gqa] fp16 (llama.cpp:2323), V transposed
 * [layer][n_embd_gqa][n_ctx] fp16 (llama.cpp:2327-2329).
 *
 * Pinned by tests/test_oracle.py::test_full_eval_matches_reference_golden (the golden logits were produced by the
 * unmodified reference) and, when oracle/_ref exists, against the reference run live.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "ggml_oracle.h"

/* from ggml_oracle.c */
int orc_mul_mat(int type, const void *w, const float *x, float *dst, int K, int M, int N);
void orc_rms_norm_mul(const float *x, const float *w, float *y, int n, float eps);
void orc_layer_norm_mul_add(const float *x, const float *w, const float *b, float *y, int n, float eps);
void orc_rope(float *x, int n_heads, int head_dim, int p, int mode, float freq_base, float freq_scale);
void orc_silu(const float *x, float *y, int n);
void orc_gelu(const float *x, float *y, int n);
void orc_attn_head_n(const float *q, const uint16_t *kcache, size_t k_stride, const uint16_t *vcache, size_t v_stride,
                     int head_dim, int T, int n_total, float kq_scale, float *out);
void orc_dequantize_row_q4_0(const void *vx, float *y, int k);
void orc_dequantize_row_q5_0(const void *vx, float *y, int k);
void orc_dequantize_row_q8_0(const void *vx, float *y, int k);
void orc_dequantize_row_q4_K(const void *vx, float *y, int k);
void orc_dequantize_row_q5_K(const void *vx, float *y, int k);
void orc_dequantize_row_q6_K(const void *vx, float *y, int k);
int orc_sizeof_block(int type);
int orc_blck_size(int type);

typedef struct { int type; int K; int M; const void *data; } orc_mat;

typedef struct {
    orc_mat wq, wk, wv, wqkv, wo, w1, w2, w3;
    const float *attn_norm, *attn_norm_b, *attn_norm2, *attn_norm2_b, *ffn_norm;
} orc_layer;

typedef struct {
    int falcon;
    int n_vocab, n_embd, n_ff, n_head, n_head_kv, n_layer, n_ctx;
    float eps, rope_base, rope_scale;
    orc_mat tok_embd, output;
    const float *out_norm, *out_norm_b;
    orc_layer *layers;
    uint16_t *kc, *vc;
    /* optional trace: if non-NULL, receives the residual stream after every layer of the LAST evaluated token,
     * [n_layer][n_embd], plus (trace_attn) the attention block's merged output [n_layer][n_embd] */
    float *trace_layer_out, *trace_attn;
    /* tensor-parallel summation mode (NOT a reference behaviour: the restatement of what ctransformers_b200's sharded engine
     * computes, csrc/engine.cu build_ops): wo / w2 are row-parallel, rank r multiplies the K range [split[r], split[r+1]) of the
     * activation as a matrix of its own (its fp32 chains start at zero at its first block), rank 0 adds the residual, and the
     * ranks' vectors are added in rank order (world 2: a single commutative fp32 add, i.e. exactly what an all-reduce gives). */
    int tp_world; int tp_wo[17], tp_w2[17];
} orc_model;

orc_model *orc_model_new(int falcon, int n_vocab, int n_embd, int n_ff, int n_head, int n_head_kv, int n_layer, int n_ctx, float eps,
                         float rope_base, float rope_scale) {
    orc_model *m = (orc_model *)calloc(1, sizeof(orc_model));
    m->falcon = falcon; m->n_vocab = n_vocab; m->n_embd = n_embd; m->n_ff = n_ff; m->n_head = n_head; m->n_head_kv = n_head_kv;
    m->n_layer = n_layer; m->n_ctx = n_ctx; m->eps = eps; m->rope_base = rope_base; m->rope_scale = rope_scale;
    m->layers = (orc_layer *)calloc((size_t)n_layer, sizeof(orc_layer));
    const size_t kv = (size_t)n_layer * n_ctx * (n_embd / n_head * n_head_kv);
    m->kc = (uint16_t *)calloc(kv, 2);
    m->vc = (uint16_t *)calloc(kv, 2);
    return m;
}
void orc_model_free(orc_model *m) { if (m) { free(m->layers); free(m->kc); free(m->vc); free(m); } }

/* slot: 0 tok_embd, 1 output, 10+ per-layer {0 wq,1 wk,2 wv,3 wqkv,4 wo,5 w1,6 w2,7 w3} */
void orc_model_set_mat(orc_model *m, int layer, int slot, int type, int K, int M, const void *data) {
    orc_mat v = {type, K, M, data};
    if (layer < 0) { if (slot == 0) m->tok_embd = v; else m->output = v; return; }
    orc_layer *L = &m->layers[layer];
    orc_mat *dst[8] = {&L->wq, &L->wk, &L->wv, &L->wqkv, &L->wo, &L->w1, &L->w2, &L->w3};
    *dst[slot] = v;
}
/* slot: 0 out_norm, 1 out_norm_b; per layer {0 attn_norm, 1 attn_norm_b, 2 attn_norm2, 3 attn_norm2_b, 4 ffn_norm} */
void orc_model_set_vec(orc_model *m, int layer, int slot, const float *data) {
    if (layer < 0) { if (slot == 0) m->out_norm = data; else m->out_norm_b = data; return; }
    orc_layer *L = &m->layers[layer];
    const float **dst[5] = {&L->attn_norm, &L->attn_norm_b, &L->attn_norm2, &L->attn_norm2_b, &L->ffn_norm};
    *dst[slot] = data;
}
int orc_model_set_tp(orc_model *m, int world, const int *wo_split, const int *w2_split) {
    if (world < 1 || world > 16) return -1;
    m->tp_world = world;
    for (int r = 0; r <= world; r++) { m->tp_wo[r] = wo_split[r]; m->tp_w2[r] = w2_split[r]; }
    return 0;
}
void orc_model_set_trace(orc_model *m, float *layer_out, float *attn) { m->trace_layer_out = layer_out; m->trace_attn = attn; }

/* ggml_get_rows on a (possibly quantized) table: ggml.c:11615-11642 */
static void get_row(const orc_mat *t, int row, float *out) {
    const int K = t->K;
    if (t->type == 0) { memcpy(out, (const float *)t->data + (size_t)row * K, (size_t)K * 4); return; }
    if (t->type == 1) { const uint16_t *h = (const uint16_t *)t->data + (size_t)row * K; for (int i = 0; i < K; i++) out[i] = orc_fp16_to_fp32(h[i]); return; }
    const char *p = (const char *)t->data + (size_t)row * (K / orc_blck_size(t->type)) * orc_sizeof_block(t->type);
    switch (t->type) {
        case 2: orc_dequantize_row_q4_0(p, out, K); break;
        case 3: orc_dequantize_row_q4_1(p, out, K); break;
        case 6: orc_dequantize_row_q5_0(p, out, K); break;
        case 7: orc_dequantize_row_q5_1(p, out, K); break;
        case 8: orc_dequantize_row_q8_0(p, out, K); break;
        case 11: orc_dequantize_row_q3_K(p, out, K); break;
        case 12: orc_dequantize_row_q4_K(p, out, K); break;
        case 13: orc_dequantize_row_q5_K(p, out, K); break;
        case 14: orc_dequantize_row_q6_K(p, out, K); break;
    }
}

/* mul_mat for one activation row; F16/F32 weights follow ggml.c:11031 with vec_dot_type F16 / F32 */
static void matvec(const orc_mat *w, const float *x, float *y) {
    if (w->type == 0) {
        for (int m = 0; m < w->M; m++) {
            const float *r = (const float *)w->data + (size_t)m * w->K; float s = 0;
            for (int i = 0; i < w->K; i++) s += r[i] * x[i];
            y[m] = s;
        }
    } else if (w->type == 1) {
        for (int m = 0; m < w->M; m++) {
            const uint16_t *r = (const uint16_t *)w->data + (size_t)m * w->K; float s = 0;
            for (int i = 0; i < w->K; i++) s += orc_fp16_to_fp32(r[i]) * orc_fp16_to_fp32(orc_fp32_to_fp16(x[i]));
            y[m] = s;
        }
    } else {
        orc_mul_mat(w->type, w->data, x, y, w->K, w->M, 1);
    }
}

/* x = all-reduce over ranks of (rank 0: x + W_0 a_0; rank r: W_r a_r), W_r = columns [split[r], split[r+1]) of w (quantized types only) */
static void matvec_row_parallel(const orc_mat *w, const float *a, float *x, int world, const int *split) {
    const int be = orc_blck_size(w->type), bb = orc_sizeof_block(w->type);
    const size_t full_row = (size_t)(w->K / be) * bb;
    float *part = (float *)malloc(sizeof(float) * w->M);
    for (int r = 0; r < world; r++) {
        const int k0 = split[r], k1 = split[r + 1], nbl = (k1 - k0) / be;
        char *sl = (char *)malloc((size_t)w->M * nbl * bb);
        for (int m = 0; m < w->M; m++) memcpy(sl + (size_t)m * nbl * bb, (const char *)w->data + (size_t)m * full_row + (size_t)(k0 / be) * bb, (size_t)nbl * bb);
        orc_mul_mat(w->type, sl, a + k0, part, k1 - k0, w->M, 1);
        for (int i = 0; i < w->M; i++) x[i] = x[i] + part[i];
        free(sl);
    }
    free(part);
}

/* One token at absolute position pos.  x: [n_embd] residual stream in/out. */
static void eval_token(orc_model *m, int token, int pos, int n_total, int want_out, float *logits, float *embd) {
    const int E = m->n_embd, H = m->n_head, HK = m->n_head_kv, hd = E / H, G = hd * HK, FF = m->n_ff, C = m->n_ctx;
    const float kq_scale = 1.0f / sqrtf((float)E / (float)H);   /* llama.cpp:2260-2264 */
    float *x = (float *)malloc(sizeof(float) * E), *nrm = (float *)malloc(sizeof(float) * E), *nrm2 = (float *)malloc(sizeof(float) * E);
    float *q = (float *)malloc(sizeof(float) * (E + 2 * G)), *att = (float *)malloc(sizeof(float) * E), *tmp = (float *)malloc(sizeof(float) * E);
    float *g = (float *)malloc(sizeof(float) * FF), *u = (float *)malloc(sizeof(float) * FF), *ao = (float *)malloc(sizeof(float) * E);
    get_row(&m->tok_embd, token, x);
    for (int il = 0; il < m->n_layer; il++) {
        const orc_layer *L = &m->layers[il];
        uint16_t *kc = m->kc + (size_t)il * C * G, *vc = m->vc + (size_t)il * C * G;
        float *k, *v;
        if (!m->falcon) {
            orc_rms_norm_mul(x, L->attn_norm, nrm, E, m->eps);
            k = q + E; v = q + E + G;
            matvec(&L->wk, nrm, k); matvec(&L->wq, nrm, q); matvec(&L->wv, nrm, v);
            orc_rope(k, HK, hd, pos, 0, m->rope_base, m->rope_scale);
            orc_rope(q, H, hd, pos, 0, m->rope_base, m->rope_scale);
        } else {
            orc_layer_norm_mul_add(x, L->attn_norm, L->attn_norm_b, nrm, E, m->eps);
            const float *in = nrm;
            if (L->attn_norm2) { orc_layer_norm_mul_add(x, L->attn_norm2, L->attn_norm2_b, nrm2, E, m->eps); in = nrm2; }
            matvec(&L->wqkv, in, q);
            k = q + (size_t)H * hd; v = k + G;
            orc_rope(q, H, hd, pos, 2, m->rope_base, m->rope_scale);
            orc_rope(k, HK, hd, pos, 2, m->rope_base, m->rope_scale);
        }
        for (int i = 0; i < G; i++) {                                     /* llama.cpp:2323-2335 */
            kc[(size_t)pos * G + i] = orc_fp32_to_fp16(k[i]);
            vc[(size_t)i * C + pos] = orc_fp32_to_fp16(v[i]);
        }
        for (int h = 0; h < H; h++) {
            const int kh = h / (H / HK);                                  /* ggml.c:11067-11069 broadcast */
            orc_attn_head_n(q + (size_t)h * hd, kc + (size_t)kh * hd, (size_t)G, vc + (size_t)kh * hd * C, (size_t)C, hd, pos + 1, n_total, kq_scale, att + (size_t)h * hd);
        }
        if (want_out && m->trace_attn) memcpy(m->trace_attn + (size_t)il * E, att, sizeof(float) * E);
        if (!m->falcon) {
            if (m->tp_world > 1) matvec_row_parallel(&L->wo, att, x, m->tp_world, m->tp_wo);
            else {
                matvec(&L->wo, att, tmp);
                for (int i = 0; i < E; i++) x[i] = tmp[i] + x[i];          /* inpFF = cur + inpSA */
            }
            orc_rms_norm_mul(x, L->ffn_norm, nrm, E, m->eps);
            matvec(&L->w3, nrm, u); matvec(&L->w1, nrm, g);
            orc_silu(g, g, FF);
            for (int i = 0; i < FF; i++) g[i] = g[i] * u[i];
            if (m->tp_world > 1) matvec_row_parallel(&L->w2, g, x, m->tp_world, m->tp_w2);
            else {
                matvec(&L->w2, g, tmp);
                for (int i = 0; i < E; i++) x[i] = tmp[i] + x[i];
            }
        } else {
            matvec(&L->wo, att, ao);                                       /* attn_out */
            matvec(&L->w3, nrm, g);                                        /* FFN reads the SAME normed input (parallel block) */
            orc_gelu(g, g, FF);
            matvec(&L->w2, g, tmp);
            for (int i = 0; i < E; i++) x[i] = (tmp[i] + ao[i]) + x[i];   /* llama.cpp:2767-2771 */
        }
        if (want_out && m->trace_layer_out) memcpy(m->trace_layer_out + (size_t)il * E, x, sizeof(float) * E);
    }
    if (want_out) {
        if (!m->falcon) orc_rms_norm_mul(x, m->out_norm, nrm, E, m->eps);
        else orc_layer_norm_mul_add(x, m->out_norm, m->out_norm_b, nrm, E, m->eps);
        if (embd) memcpy(embd, nrm, sizeof(float) * E);
        if (logits) matvec(&m->output, nrm, logits);
    }
    free(x); free(nrm); free(nrm2); free(q); free(att); free(tmp); free(g); free(u); free(ao);
}

/* llama_eval: n tokens from position n_past; logits/embd of the last one (llama.cpp:2949-2968) */
int orc_eval(orc_model *m, const int *tokens, int n, int n_past, float *logits, float *embd) {
    if (n_past + n > m->n_ctx) return -1;
    for (int i = 0; i < n; i++) {
        if (tokens[i] < 0 || tokens[i] >= m->n_vocab) return -2;
        eval_token(m, tokens[i], n_past + i, n_past + n, i == n - 1, logits, embd);
    }
    return 0;
}

/* llama_eval with the context flag logits_all (llama.cpp:2949-2960): the same graph, with the output row of every token of
 * the call copied out.  Token i's logits go to logits[i * n_vocab]; embd gets the last token's result_norm row. */
int orc_eval_rows(orc_model *m, const int *tokens, int n, int n_past, float *logits, float *embd) {
    if (n_past + n > m->n_ctx) return -1;
    for (int i = 0; i < n; i++) {
        if (tokens[i] < 0 || tokens[i] >= m->n_vocab) return -2;
        eval_token(m, tokens[i], n_past + i, n_past + n, 1, logits + (size_t)i * m->n_vocab, i == n - 1 ? embd : NULL);
    }
    return 0;
}
