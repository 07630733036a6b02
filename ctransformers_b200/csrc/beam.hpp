// Beam search selection on the host: the reference's llama_beam_search (models/ggml/llama.cpp:4334-4579) step by step.
//
// Every float that ranks beams is computed here, on the host, from the fetched logits rows, in the reference's order: the
// row's maximum (std::max_element), the normaliser 1 / (sequential fp32 sum of expf(l - max) in vocabulary order) with the
// host libm's expf, each candidate's probability normaliser * expf(l - max), and the beam's p times it.  The candidates and
// the next beams are min-heaps built with the same std heap calls in the same order, so their array order — which decides
// ties, the renormalising sum and the top beam — is the reference's.
#pragma once
#include <algorithm>
#include <cmath>
#include <numeric>
#include <stdexcept>
#include <vector>

namespace ctb {

// One beam as the selection sees it.  parent: index of the beam it came from in the previous step's array; token: the token it
// added, -1 for an eob beam carried over unevaluated.
struct BeamCand {
  float p;
  bool eob;
  int parent, token;
};

// The reference's ordering of beams (llama_beam::operator<): by p, and at equal p the eob beam is the larger.
inline bool beam_less(const BeamCand& a, const BeamCand& b) { return a.p < b.p || (a.p == b.p && a.eob < b.eob); }

// Index of the top beam: the first maximum under beam_less (std::max_element).
inline size_t beam_top(const std::vector<BeamCand>& beams) {
  return (size_t)(std::max_element(beams.begin(), beams.end(), beam_less) - beams.begin());
}

struct BeamToken { int id; float logit; };

// The k largest logits of a row (llama_logit_info::top_k): ids 0 .. k-1 seed a min-heap; a later id replaces the heap's front
// only when its logit is strictly larger.  Returned in heap array order.
inline std::vector<BeamToken> beam_top_k(const float* row, int n_vocab, size_t k) {
  const auto comp = [](const BeamToken& a, const BeamToken& b) { return a.logit > b.logit; };
  const int k_min = std::min((int)k, n_vocab);
  std::vector<BeamToken> heap;
  heap.reserve(k_min);
  for (int id = 0; id < k_min; ++id) heap.push_back({id, row[id]});
  std::make_heap(heap.begin(), heap.end(), comp);
  for (int id = k_min; id < n_vocab; ++id) {
    if (heap.front().logit < row[id]) {
      std::pop_heap(heap.begin(), heap.end(), comp);
      heap.back() = {id, row[id]};
      std::push_heap(heap.begin(), heap.end(), comp);
    }
  }
  return heap;
}

// Adds the continuations of beam `parent` (or the beam itself when it is eob) to `next`, the min-heap by p of the next step's
// beams (llama_beam_search_data::fill_next_beams_by_top_probabilities).  row: the beam's logits (unused for an eob beam).
// `next` is not emptied between steps: its old entries have p = 0 and are replaced while the front's p is 0.  The reference
// reads past its candidates when a continuation's p is 0 there too; that is an error here.
inline void beam_fill(size_t n_beams, const BeamCand& beam, int parent, const float* row, int n_vocab, std::vector<BeamCand>& next) {
  const auto comp = [](const BeamCand& a, const BeamCand& b) { return a.p > b.p; };
  if (beam.eob) {
    const BeamCand carried{beam.p, true, parent, -1};
    if (next.size() < n_beams) {
      next.push_back(carried);
      if (next.size() == n_beams) std::make_heap(next.begin(), next.end(), comp);
    } else if (next.front().p < carried.p) {
      std::pop_heap(next.begin(), next.end(), comp);
      next.back() = carried;
      std::push_heap(next.begin(), next.end(), comp);
    }
    return;
  }
  const float max_l = *std::max_element(row, row + n_vocab);
  const float normalizer = 1.0f / std::accumulate(row, row + n_vocab, 0.0f, [=](float sum, float l) { return sum + std::exp(l - max_l); });
  const std::vector<BeamToken> top = beam_top_k(row, n_vocab, n_beams);
  const auto child = [&](size_t i) { return BeamCand{beam.p * (normalizer * std::exp(top[i].logit - max_l)), false, parent, top[i].id}; };
  size_t i = 0;
  if (next.size() < n_beams) {
    for (; next.size() < n_beams; ++i) next.push_back(child(i));
    std::make_heap(next.begin(), next.end(), comp);
  } else {
    for (; next.front().p == 0.0f; ++i) {
      if (i >= top.size())
        throw std::domain_error("beam search: every continuation's probability underflows to 0 (p of the beam " + std::to_string(beam.p) + ")");
      std::pop_heap(next.begin(), next.end(), comp);
      next.back() = child(i);
      std::push_heap(next.begin(), next.end(), comp);
    }
  }
  for (; i < n_beams; ++i) {
    const BeamCand c = child(i);
    if (next.front().p < c.p) {
      std::pop_heap(next.begin(), next.end(), comp);
      next.back() = c;
      std::push_heap(next.begin(), next.end(), comp);
    }
  }
}

// One selection step over the beams of a step (after their eob flags are set): `next` holds the previous step's beams (empty at
// the first step), zeroed and refilled; then the new beams are renormalised to sum to 1 (a sequential fp32 sum in array order).
// rows[i]: the logits of beams[i] (n_vocab floats; unused for eob beams).  Returns the new beams in heap array order.
// An old entry that no beam displaced means a continuation's p was 0, which the reference does not define: an error here.
inline std::vector<BeamCand> beam_step(size_t n_beams, const std::vector<BeamCand>& beams, std::vector<BeamCand> next, const float* const* rows, int n_vocab) {
  for (BeamCand& b : next) b = BeamCand{0.0f, false, -1, -1};
  for (size_t i = 0; i < beams.size(); ++i) beam_fill(n_beams, beams[i], (int)i, rows[i], n_vocab, next);
  for (const BeamCand& b : next)
    if (b.parent < 0) throw std::domain_error("beam search: a continuation's probability underflows to 0");
  const float inv_sum = 1.0f / std::accumulate(next.begin(), next.end(), 0.0f, [](float sum, const BeamCand& b) { return sum + b.p; });
  for (BeamCand& b : next) b.p *= inv_sum;
  return next;
}

}  // namespace ctb
