// Grammar-constrained sampling, device half: k_grammar_mask writes, for every constrained row and every token, the row's logit
// after its repetition penalty (sample_gpu.cuh sg_penalised) where the grammar allows the token and -inf where it does not: what
// llama_sample_grammar (models/ggml/llama.cpp:4085-4123) leaves after llama_sample_repetition_penalty.  The rows go to a scratch
// buffer [rows][n_vocab]; k_sample_topk (penalty 1, no window) and the host sampler then run on it unchanged.
//
// One thread per (row, token).  The thread decodes its token's piece after the row's partial UTF-8 sequence (decode_utf8,
// 3450-3504) and searches the row's stacks depth first for one that accepts the code points (the per-candidate reading of
// llama_grammar_reject_candidates, 3678-3751: a token is allowed iff some stack accepts it).  A stack is a chain of immutable
// nodes {element, parent}: the row's stacks arrive as nodes, and a thread pushes its own into a small pool, so popping and
// backtracking only move an index.  The pool, the work list, the decoded length and the number of steps are bounded; a thread
// that reaches a bound marks its row, and the host recomputes that row's mask (grammar.hpp).  A bound never makes a wrong mask.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "sample_gpu.cuh"

namespace ctb {

constexpr int GM_THREADS = 256;
constexpr int GM_MAX_CP = 48;       // code points of one decoded piece
constexpr int GM_POOL = 96;         // nodes a thread may push at once
constexpr int GM_WORK = 48;         // pending (stack, position) pairs
constexpr int GM_MAX_STEPS = 4096;  // work items one thread may visit
constexpr int GM_ROW_INTS = 10;
__host__ __device__ inline int gm_words(int n_vocab) { return (n_vocab + 31) / 32; }

// One row of a launch, as ints of the argument block:
//   slot        whose kept logits (row `slot` of logits)
//   rule_base   where the row's grammar's rule offsets start in rule_off (absolute element indices)
//   head0, n_heads   the row's stack tops: heads[head0 ..), node indices (-1: an empty stack)
//   pu_value, pu_n   the pending partial UTF-8 sequence
//   eos_ok      some stack is empty
//   last0, n_last    the repetition window: last_tokens[last0 ..)
//   penalty     float bits
struct GmArgs {
  const float* logits;        // [slots][n_vocab]
  const int* rows;            // [R][GM_ROW_INTS]
  const uint32_t* elems;      // [type, value] pairs of every grammar of the launch
  const int* rule_off;
  const int* nodes;           // [element, parent] pairs; parent -1 is the stack's bottom
  const int* heads;
  const int* last_tokens;
  const int* piece_off;       // [n_vocab + 1] into piece_bytes (each piece cut at its first NUL)
  const uint8_t* piece_bytes;
  float* out;                 // [R][n_vocab]
  int* stats;                 // [R][2]: allowed tokens, a bound was reached
  unsigned* bits;             // [R][gm_words(n_vocab)]: bit t % 32 of word t / 32 set where token t is allowed
  int n_vocab, eos;
};

__device__ __forceinline__ bool gm_end(const uint32_t* el, int e) { const uint32_t t = el[2 * e]; return t == 0u || t == 1u; }

// llama_grammar_match_char; *after: the element after the class
__device__ __forceinline__ bool gm_match(const uint32_t* el, int e, uint32_t chr, int* after) {
  bool found = false;
  const bool pos = el[2 * e] == 3u;
  do {
    if (el[2 * (e + 1)] == 5u) { found = found || (el[2 * e + 1] <= chr && chr <= el[2 * (e + 1) + 1]); e += 2; }
    else { found = found || el[2 * e + 1] == chr; e += 1; }
  } while (el[2 * e] == 6u);
  *after = e;
  return found == pos;
}

// llama_grammar_match_partial_char
__device__ __forceinline__ bool gm_match_partial(const uint32_t* el, int e, uint32_t value, int n_remain) {
  const bool pos = el[2 * e] == 3u;
  if (n_remain < 0 || (n_remain == 1 && value < 2)) return false;
  uint32_t lo = value << (n_remain * 6);
  const uint32_t hi = lo | ((1u << (n_remain * 6)) - 1);
  if (lo == 0) { if (n_remain == 2) lo = 1u << 11; else if (n_remain == 3) lo = 1u << 16; }
  do {
    if (el[2 * (e + 1)] == 5u) {
      if (el[2 * e + 1] <= hi && lo <= el[2 * (e + 1) + 1]) return pos;
      e += 2;
    } else {
      if (lo <= el[2 * e + 1] && el[2 * e + 1] <= hi) return pos;
      e += 1;
    }
  } while (el[2 * e] == 6u);
  return !pos;
}

// Whether the row's stacks allow token t: 1 allowed, 0 rejected, -1 a bound was reached.
__device__ int gm_allowed(const GmArgs& a, const int* row, int t) {
  if (t == a.eos) return row[6];
  const int p0 = __ldg(a.piece_off + t), p1 = __ldg(a.piece_off + t + 1);
  if (p1 == p0) return 0;   // empty piece (or one that starts with NUL)
  // decode_utf8 after the row's partial sequence
  uint32_t cps[GM_MAX_CP];
  int ncp = 0;
  uint32_t v = (uint32_t)row[4];
  int rem = row[5];
  const int rem0 = rem;
  int i = p0;
  while (i < p1 && rem > 0) {
    const uint32_t b = __ldg(a.piece_bytes + i);
    if ((b >> 6) != 2u) return 0;
    v = (v << 6) + (b & 0x3Fu);
    i++;
    rem--;
  }
  // the reference ends a candidate's code points at the first 0 (its terminator, llama.cpp:3692, 3703): an overlong-encoded NUL
  // ends the piece for the mask there, while the rest is still decoded for its validity and the partial state it leaves
  bool ended = false;
  if (rem0 > 0 && rem == 0) {
    if (v == 0) ended = true;
    else cps[ncp++] = v;
  }
  while (i < p1) {
    const uint32_t b = __ldg(a.piece_bytes + i);
    const uint32_t hb = b >> 4;
    rem = hb < 8u ? 0 : hb < 12u ? -1 : hb < 14u ? 1 : hb == 14u ? 2 : 3;
    if (rem < 0) return 0;
    v = b & ((1u << (7 - rem)) - 1);
    i++;
    while (i < p1 && rem > 0) { v = (v << 6) + (__ldg(a.piece_bytes + i) & 0x3Fu); i++; rem--; }
    if (rem == 0 && !ended) {
      if (v == 0) { ended = true; continue; }
      if (ncp == GM_MAX_CP) return -1;
      cps[ncp++] = v;
    }
  }
  // every stack accepts a piece that ends on a whole code point once its characters have matched (advance_stack leaves at least
  // one stack); with a partial sequence pending, the stack's next class must admit a completion
  const uint32_t* el = a.elems;
  const int* roff = a.rule_off + row[1];
  int pe[GM_POOL], pp[GM_POOL];   // the thread's nodes: index k is node -(k + 2)
  int wn[GM_WORK], wc[GM_WORK], wm[GM_WORK];   // work: stack top, code point index, pool size when pushed
  int np = 0, nw = 0, steps = 0;
  for (int h = row[3] - 1; h >= 0; h--) {
    if (nw == GM_WORK) return -1;
    wn[nw] = __ldg(a.heads + row[2] + h); wc[nw] = 0; wm[nw] = 0; nw++;
  }
  while (nw > 0) {
    if (++steps > GM_MAX_STEPS) return -1;
    nw--;
    const int n = wn[nw], ci = wc[nw];
    np = wm[nw];   // nodes pushed after this item were only referenced by items already done
    if (ci == ncp && rem == 0) return 1;
    if (n == -1) continue;   // an empty stack accepts only the end of the piece
    const int e = n >= 0 ? __ldg(a.nodes + 2 * n) : pe[-n - 2];
    const int parent = n >= 0 ? __ldg(a.nodes + 2 * n + 1) : pp[-n - 2];
    const uint32_t type = el[2 * e];
    if (type == 2u) {   // rule reference: one stack per alternative (llama_grammar_advance_stack)
      int base = parent;
      if (!gm_end(el, e + 1)) {
        if (np == GM_POOL) return -1;
        pe[np] = e + 1; pp[np] = parent; base = -(np + 2); np++;
      }
      const int r = (int)el[2 * e + 1];
      int sub = roff[r];
      for (;;) {
        int top = base;
        if (!gm_end(el, sub)) {
          if (np == GM_POOL) return -1;
          pe[np] = sub; pp[np] = base; top = -(np + 2); np++;
        }
        if (nw == GM_WORK) return -1;
        wn[nw] = top; wc[nw] = ci; wm[nw] = np; nw++;
        while (!gm_end(el, sub)) sub++;
        if (el[2 * sub] != 1u) break;
        sub++;
      }
      continue;
    }
    if (ci == ncp) {   // a partial sequence is pending at a character class
      if (gm_match_partial(el, e, v, rem)) return 1;
      continue;
    }
    int after = 0;
    if (!gm_match(el, e, cps[ci], &after)) continue;
    int top = parent;
    if (!gm_end(el, after)) {
      if (np == GM_POOL) return -1;
      pe[np] = after; pp[np] = parent; top = -(np + 2); np++;
    }
    if (nw == GM_WORK) return -1;
    wn[nw] = top; wc[nw] = ci + 1; wm[nw] = np; nw++;
  }
  return 0;
}

static __global__ void __launch_bounds__(GM_THREADS) k_grammar_mask(const GmArgs a) {
  const int r = blockIdx.y;
  const int t = blockIdx.x * GM_THREADS + threadIdx.x;
  const int* row = a.rows + (size_t)r * GM_ROW_INTS;
  int ok = 0, bound = 0;
  if (t < a.n_vocab) {
    const float penalty = __int_as_float(row[9]);
    const float v = sg_penalised(a.logits + (size_t)row[0] * a.n_vocab, t, a.last_tokens + row[7], row[8], penalty);
    const int allowed = gm_allowed(a, row, t);
    ok = allowed == 1;
    bound = allowed < 0;
    a.out[(size_t)r * a.n_vocab + t] = ok ? v : __int_as_float((int)0xff800000);   // -inf
  }
  const unsigned okb = __ballot_sync(0xffffffffu, ok);
  const unsigned any_bound = __ballot_sync(0xffffffffu, bound);
  if ((threadIdx.x & 31) == 0 && t < a.n_vocab) {
    a.bits[(size_t)r * gm_words(a.n_vocab) + t / 32] = okb;
    if (okb) atomicAdd(a.stats + 2 * r, __popc(okb));
    if (any_bound) atomicOr(a.stats + 2 * r + 1, 1);
  }
}

}  // namespace ctb
