/*
 * logits_all_oracle.c — TEST INFRASTRUCTURE ONLY: orc_eval_all on top of the whole-model oracle, without changing it.
 *
 * The reference's llama_eval with the context flag logits_all (models/ggml/llama.cpp:2949-2960) runs the same graph and copies
 * the output row of every token of the call, not only the last one's.  orc_eval_all is orc_eval (oracle/llama_oracle.c) with
 * want_out set for every token: token i's logits go to logits[i * n_vocab]; embd gets the last token's result_norm row.
 *
 * This file is one translation unit with the oracle it extends (eval_token is static there): compiled as it is, the plain
 * oracle (oracle/ggml_oracle.c + oracle/llama_oracle.c, as tests/head_dims_oracle.c combines them); with
 * -DORACLE_TU='"<file>"' one of the per-type oracles under tests/ (q3k_oracle.c, q41_q51_oracle.c, head_dims_oracle.c), which
 * include both themselves.  tests/logits_all_cases.py builds it.
 */
#ifdef ORACLE_TU
#include ORACLE_TU
#else
#include "../oracle/ggml_oracle.c"
#include "../oracle/llama_oracle.c"
#endif

int orc_eval_all(orc_model *m, const int *tokens, int n, int n_past, float *logits, float *embd) {
    if (n_past + n > m->n_ctx) return -1;
    for (int i = 0; i < n; i++) {
        if (tokens[i] < 0 || tokens[i] >= m->n_vocab) return -2;
        eval_token(m, tokens[i], n_past + i, n_past + n, 1, logits + (size_t)i * m->n_vocab, i == n - 1 ? embd : NULL);
    }
    return 0;
}
