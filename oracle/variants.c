/*
 * variants.c — TEST INFRASTRUCTURE ONLY (same rules as ggml_oracle.c): the setters of the forms the reference does NOT use, for
 * the tests that show the stored reference results tell those forms apart.  Each variant starts at 0, the reference's
 * arithmetic; the values are described where each is read.
 */
extern int orc_q3k_variant, orc_q1_variant, orc_hd_variant;

void orc_q3k_set_variant(int v) { orc_q3k_variant = v; }   /* q3k_oracle.c: orc_vec_dot_q3_K_q8_K   */
void orc_q1_set_variant(int v) { orc_q1_variant = v; }     /* q41_q51_oracle.c: Q1_* bits            */
void orc_hd_set_variant(int v) { orc_hd_variant = v; }     /* ggml_oracle.c: orc_attn_head_n's K·q dot */
