// Host-side token sampler behind ctransformers_llm_sample.
//
// Same chain, same comparators and the same libstdc++ primitives as the reference so that a seeded draw
// returns the same token: repetition penalty → top-k → top-p → temperature → softmax → discrete draw
// (reference: models/llms/llama.cc:53-84; models/ggml/llama.cpp:3805-3830 softmax, 3832-3857 top-k,
//  3859-3890 top-p, 4013-4023 temperature, 4025-4055 repetition penalty, 4281-4302 draw).
#pragma once
#include <algorithm>
#include <cmath>
#include <random>
#include <vector>

namespace ctb {

struct Candidate { int id; float logit; float p; };

inline void softmax_sorted(std::vector<Candidate>& c, size_t& n, bool& sorted) {
  auto by_logit = [](const Candidate& a, const Candidate& b) { return a.logit > b.logit; };
  if (!sorted) { std::sort(c.begin(), c.begin() + n, by_logit); sorted = true; }
  const float top = c[0].logit;
  float total = 0.0f;
  for (size_t i = 0; i < n; i++) { float p = expf(c[i].logit - top); c[i].p = p; total += p; }
  for (size_t i = 0; i < n; i++) c[i].p /= total;
}

// top-k → top-p → temperature → softmax → draw over candidates whose repetition penalty has been applied already
inline int sample_candidates(std::vector<Candidate>& c, int top_k, float top_p, float temperature, std::mt19937& rng) {
  size_t n = c.size();
  bool sorted = false;
  auto by_logit = [](const Candidate& a, const Candidate& b) { return a.logit > b.logit; };
  {  // top-k, min_keep = 1
    int k = std::min(std::max(top_k, 1), (int)n);
    if (!sorted) {
      if (k == (int)n) std::sort(c.begin(), c.begin() + n, by_logit);
      else std::partial_sort(c.begin(), c.begin() + k, c.begin() + n, by_logit);
      sorted = true;
    }
    n = (size_t)k;
  }
  if (top_p < 1.0f) {  // top-p, min_keep = 1
    softmax_sorted(c, n, sorted);
    float cum = 0.0f;
    size_t keep = n;
    for (size_t i = 0; i < n; i++) {
      cum += c[i].p;
      if (cum >= top_p && i + 1 >= 1) { keep = i + 1; break; }
    }
    n = keep;
  }
  for (size_t i = 0; i < n; i++) c[i].logit /= temperature;
  softmax_sorted(c, n, sorted);
  std::vector<float> probs;
  probs.reserve(n);
  for (size_t i = 0; i < n; i++) probs.push_back(c[i].p);
  std::discrete_distribution<> dist(probs.begin(), probs.end());
  return c[dist(rng)].id;
}

inline int sample_token(const float* logits, int n_vocab, const int* last, int n_last, int top_k, float top_p,
                        float temperature, float penalty, std::mt19937& rng) {
  std::vector<Candidate> c;
  c.reserve(n_vocab);
  for (int i = 0; i < n_vocab; i++) c.push_back(Candidate{i, logits[i], 0.0f});
  if (n_last > 0 && penalty != 1.0f) {
    for (size_t i = 0; i < c.size(); i++) {
      if (std::find(last, last + n_last, c[i].id) == last + n_last) continue;
      if (c[i].logit <= 0) c[i].logit *= penalty; else c[i].logit /= penalty;
    }
  }
  return sample_candidates(c, top_k, top_p, temperature, rng);
}

// The candidates the device-side top-k returned (sample_gpu.cuh): every logit >= the k-th largest, penalty applied.  Usable
// only when the cut is unambiguous: exactly k of them (no tie at the threshold) and no two equal logits (std::partial_sort
// leaves the order of equal elements unspecified; then only the sort over ALL candidates reproduces the reference).
inline bool device_candidates_usable(const int* ids, const float* logits, int count, int top_k, int n_vocab, std::vector<Candidate>& c) {
  const int k = std::min(std::max(top_k, 1), n_vocab);
  if (count != k) return false;
  c.clear();
  for (int i = 0; i < count; i++) c.push_back(Candidate{ids[i], logits[i], 0.0f});
  std::sort(c.begin(), c.end(), [](const Candidate& a, const Candidate& b) { return a.id < b.id; });   // the order they have in the full list
  for (int i = 0; i < count; i++)
    for (int j = i + 1; j < count; j++)
      if (c[i].logit == c[j].logit) return false;
  return true;
}

// The draws the greedy shortcut answers: one candidate survives top-k, so top-p / temperature / the draw cannot change it
// (llama.cpp:3832-3857, 4215-4240).
inline bool sample_is_greedy(int top_k, float penalty, int n_last) { return top_k == 1 && (penalty == 1.0f || n_last <= 0); }

// The sampler chain for logits that are still on the device (ctransformers_llm_sample before anybody asked for a host view):
// penalty + top-k run on the device and only the candidates come back; the host finishes with the same code as sample_token.
//   pick()                                   the device's greedy pick when it is the only largest logit, else < 0
//   topk(last, n_last, penalty, k, ids, lg)  the device candidates (Engine::topk_candidates): their count, < 0 when the device
//                                            cannot answer
//   all()                                    the full logits on the host, as a std::vector<float>
// used_device: whether the device answered (false: the host sampler ran on all()).
template <class Pick, class TopK, class All>
int sample_lazy(int n_vocab, const int* last, int n_last, int top_k, float top_p, float temperature, float penalty, std::mt19937& rng,
                bool& used_device, Pick&& pick, TopK&& topk, All&& all) {
  used_device = true;
  if (sample_is_greedy(top_k, penalty, n_last)) {
    // Equal maxima fall through (std::partial_sort's choice among equals is the reference's).
    const int p = pick();
    if (p >= 0) return p;
  }
  int ids[256];
  float lg[256];
  const int count = topk(last, n_last, penalty, top_k, ids, lg);
  std::vector<Candidate> c;
  if (count > 0 && device_candidates_usable(ids, lg, count, top_k, n_vocab, c)) return sample_candidates(c, top_k, top_p, temperature, rng);
  // ambiguous cut (equal logits, NaN): the reference's own sort over all candidates decides — host path on a private copy
  used_device = false;
  const std::vector<float> v = all();
  return sample_token(v.data(), n_vocab, last, n_last, top_k, top_p, temperature, penalty, rng);
}

}  // namespace ctb
