// Grammar-constrained sampling, host half: the GBNF parser, the grammar state, accepting a token, and the mask of the tokens a
// state allows.
//
// Restates, without copying, the reference's grammar_parser::parse (models/submodules/llama.cpp/common/grammar-parser.cpp) and its
// grammar functions in models/ggml/llama.cpp: decode_utf8 (3450-3504), llama_grammar_match_char / match_partial_char (3517-3588),
// llama_grammar_advance_stack (3593-3644), llama_grammar_accept (3650-3676), llama_grammar_reject_candidates (3678-3751),
// llama_grammar_init (3757-3795), llama_sample_grammar (4085-4123) and llama_grammar_accept_token (4304-4328).
//
// An element is {type, value} with the types of llama.h:175-195.  The rules live in one flat array (rule r is elems[off[r] ..
// off[r + 1]), ending with END), and a stack holds element indices into it, bottom first, never pointers: the same arrays go to
// the device (grammar_gpu.cuh).
#pragma once
#include <algorithm>
#include <cstdint>
#include <map>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

namespace ctb {

enum GType : uint32_t { G_END = 0, G_ALT = 1, G_RULE_REF = 2, G_CHAR = 3, G_CHAR_NOT = 4, G_CHAR_RNG_UPPER = 5, G_CHAR_ALT = 6 };
struct GElem { uint32_t type, value; };

// A refused grammar text: what the parser expected, and the byte offset where it stopped.
struct GrammarError : std::runtime_error {
  long pos;
  GrammarError(const std::string& m, long p) : std::runtime_error(m), pos(p) {}
};

struct Grammar {
  std::vector<GElem> elems;   // every rule, one after another
  std::vector<int> off;       // rule r: elems[off[r] .. off[r + 1])
  std::vector<std::pair<std::string, uint32_t>> symbols;   // name -> id, in id order (ids are given in order of first appearance)
  uint32_t root = 0;
  int n_rules() const { return (int)off.size() - 1; }
  bool end_of_seq(int e) const { return elems[e].type == G_END || elems[e].type == G_ALT; }
};

// ---------------------------------------------------------------------------------------------------------------------------
// The parser (grammar_parser::parse).  Every error the reference prints becomes a GrammarError with the same words.
namespace gparse {

struct State {
  const char* src;
  std::map<std::string, uint32_t> ids;
  std::vector<std::vector<GElem>> rules;
  GrammarError err(const std::string& what, const char* at) const {
    std::string rest(at);
    if (rest.size() > 24) rest = rest.substr(0, 24) + "...";
    return GrammarError(what + " at '" + rest + "'", (long)(at - src));
  }
};

// the parser's own UTF-8 reading: no validation, stops at a NUL
inline std::pair<uint32_t, const char*> utf8(const char* s) {
  static const int len_of[] = {1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 2, 2, 3, 4};
  const uint8_t b = (uint8_t)*s;
  const int len = len_of[b >> 4];
  uint32_t v = b & ((1u << (8 - len)) - 1);
  const char* end = s + len;
  const char* p = s + 1;
  for (; p < end && *p; p++) v = (v << 6) + ((uint8_t)*p & 0x3F);
  return {v, p};
}

inline uint32_t symbol(State& st, const std::string& name) {
  const uint32_t next = (uint32_t)st.ids.size();
  return st.ids.insert({name, next}).first->second;
}
inline uint32_t new_symbol(State& st, const std::string& base) {
  const uint32_t next = (uint32_t)st.ids.size();
  st.ids[base + '_' + std::to_string(next)] = next;
  return next;
}
inline void put_rule(State& st, uint32_t id, const std::vector<GElem>& r) {
  if (st.rules.size() <= id) st.rules.resize(id + 1);
  st.rules[id] = r;
}
inline bool word_char(char c) { return (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || c == '-' || (c >= '0' && c <= '9'); }

inline std::pair<uint32_t, const char*> hex(State& st, const char* s, int n) {
  const char* p = s;
  const char* end = s + n;
  uint32_t v = 0;
  for (; p < end && *p; p++) {
    v <<= 4;
    const char c = *p;
    if (c >= 'a' && c <= 'f') v += c - 'a' + 10;
    else if (c >= 'A' && c <= 'F') v += c - 'A' + 10;
    else if (c >= '0' && c <= '9') v += c - '0';
    else break;
  }
  if (p != end) throw st.err("expecting " + std::to_string(n) + " hex chars", s);
  return {v, p};
}

inline const char* space(const char* s, bool newline_ok) {
  const char* p = s;
  while (*p == ' ' || *p == '\t' || *p == '#' || (newline_ok && (*p == '\r' || *p == '\n'))) {
    if (*p == '#') while (*p && *p != '\r' && *p != '\n') p++;
    else p++;
  }
  return p;
}

inline const char* name_end(State& st, const char* s) {
  const char* p = s;
  while (word_char(*p)) p++;
  if (p == s) throw st.err("expecting name", s);
  return p;
}

inline std::pair<uint32_t, const char*> one_char(State& st, const char* s) {
  if (*s == '\\') {
    switch (s[1]) {
      case 'x': return hex(st, s + 2, 2);
      case 'u': return hex(st, s + 2, 4);
      case 'U': return hex(st, s + 2, 8);
      case 't': return {'\t', s + 2};
      case 'r': return {'\r', s + 2};
      case 'n': return {'\n', s + 2};
      case '\\': case '"': case '[': case ']': return {(uint32_t)(uint8_t)s[1], s + 2};
      default: throw st.err("unknown escape", s);
    }
  }
  if (*s) return utf8(s);
  throw st.err("unexpected end of input", s);
}

const char* alternates(State& st, const char* s, const std::string& name, uint32_t id, bool nested);

inline const char* sequence(State& st, const char* s, const std::string& name, std::vector<GElem>& out, bool nested) {
  size_t last = out.size();
  const char* p = s;
  while (*p) {
    if (*p == '"') {   // literal
      p++;
      last = out.size();
      while (*p != '"') {
        auto c = one_char(st, p);
        p = c.second;
        out.push_back({G_CHAR, c.first});
      }
      p = space(p + 1, nested);
    } else if (*p == '[') {   // character class
      p++;
      uint32_t first = G_CHAR;
      if (*p == '^') { p++; first = G_CHAR_NOT; }
      last = out.size();
      while (*p != ']') {
        auto c = one_char(st, p);
        p = c.second;
        out.push_back({last < out.size() ? (uint32_t)G_CHAR_ALT : first, c.first});
        if (p[0] == '-' && p[1] != ']') {
          auto e = one_char(st, p + 1);
          p = e.second;
          out.push_back({G_CHAR_RNG_UPPER, e.first});
        }
      }
      p = space(p + 1, nested);
    } else if (word_char(*p)) {   // rule reference
      const char* e = name_end(st, p);
      const uint32_t ref = symbol(st, std::string(p, e - p));
      p = space(e, nested);
      last = out.size();
      out.push_back({G_RULE_REF, ref});
    } else if (*p == '(') {   // group: a generated rule
      p = space(p + 1, true);
      const uint32_t sub = new_symbol(st, name);
      p = alternates(st, p, name, sub, true);
      last = out.size();
      out.push_back({G_RULE_REF, sub});
      if (*p != ')') throw st.err("expecting ')'", p);
      p = space(p + 1, nested);
    } else if (*p == '*' || *p == '+' || *p == '?') {   // S* -> S' ::= S S' |   S+ -> S' ::= S S' | S   S? -> S' ::= S |
      if (last == out.size()) throw st.err("expecting preceeding item to */+/?", p);
      const uint32_t sub = new_symbol(st, name);
      std::vector<GElem> r(out.begin() + last, out.end());
      if (*p != '?') r.push_back({G_RULE_REF, sub});
      r.push_back({G_ALT, 0});
      if (*p == '+') r.insert(r.end(), out.begin() + last, out.end());
      r.push_back({G_END, 0});
      put_rule(st, sub, r);
      out.resize(last);
      out.push_back({G_RULE_REF, sub});
      p = space(p + 1, nested);
    } else {
      break;
    }
  }
  return p;
}

inline const char* alternates(State& st, const char* s, const std::string& name, uint32_t id, bool nested) {
  std::vector<GElem> r;
  const char* p = sequence(st, s, name, r, nested);
  while (*p == '|') {
    r.push_back({G_ALT, 0});
    p = space(p + 1, true);
    p = sequence(st, p, name, r, nested);
  }
  r.push_back({G_END, 0});
  put_rule(st, id, r);
  return p;
}

inline const char* rule(State& st, const char* s) {
  const char* e = name_end(st, s);
  const char* p = space(e, false);
  const std::string name(s, e - s);
  const uint32_t id = symbol(st, name);
  if (!(p[0] == ':' && p[1] == ':' && p[2] == '=')) throw st.err("expecting ::=", p);
  p = space(p + 3, true);
  p = alternates(st, p, name, id, false);
  if (*p == '\r') p += p[1] == '\n' ? 2 : 1;
  else if (*p == '\n') p++;
  else if (*p) throw st.err("expecting newline or end", p);
  return space(p, true);
}

}  // namespace gparse

// Parse GBNF text.  Beyond the reference's syntax errors it refuses, before anything uses the rules: a missing `root`, a rule
// that is referenced but never defined, and left recursion among the rules root reaches (llama_grammar_advance_stack would
// recurse without end).
inline Grammar grammar_parse(const char* text) {
  gparse::State st{text, {}, {}};
  const char* p = gparse::space(text, true);
  while (*p) p = gparse::rule(st, p);
  Grammar g;
  g.symbols.assign(st.ids.begin(), st.ids.end());
  std::sort(g.symbols.begin(), g.symbols.end(), [](const auto& a, const auto& b) { return a.second < b.second; });
  const auto root = st.ids.find("root");
  if (root == st.ids.end()) throw GrammarError("grammar does not contain a 'root' rule", (long)(p - text));
  g.root = root->second;
  const size_t n = st.ids.size();
  st.rules.resize(std::max(st.rules.size(), n));
  for (const auto& s : g.symbols)
    if (st.rules[s.second].empty()) throw GrammarError("undefined rule '" + s.first + "'", (long)(p - text));
  g.off.push_back(0);
  for (const auto& r : st.rules) {
    g.elems.insert(g.elems.end(), r.begin(), r.end());
    g.off.push_back((int)g.elems.size());
  }
  // nullable rules (some alternative of nothing but nullable references), then the left-corner graph over them
  std::vector<char> nullable(n, 0);
  for (bool changed = true; changed;) {
    changed = false;
    for (size_t r = 0; r < n; r++) {
      if (nullable[r]) continue;
      bool all = true;
      for (int e = g.off[r]; e < g.off[r + 1]; e++) {
        const GElem x = g.elems[e];
        if (x.type == G_END || x.type == G_ALT) {
          if (all) { nullable[r] = 1; changed = true; break; }
          all = true;
        } else if (x.type != G_RULE_REF || !nullable[x.value]) {
          all = false;
        }
      }
    }
  }
  std::vector<std::vector<uint32_t>> left(n), refs(n);
  for (size_t r = 0; r < n; r++) {
    bool lead = true;
    for (int e = g.off[r]; e < g.off[r + 1]; e++) {
      const GElem x = g.elems[e];
      if (x.type == G_END || x.type == G_ALT) { lead = true; continue; }
      if (x.type == G_RULE_REF) {
        refs[r].push_back(x.value);
        if (lead) left[r].push_back(x.value);
        lead = lead && nullable[x.value];
      } else {
        lead = false;
      }
    }
  }
  std::vector<char> reach(n, 0);
  std::vector<uint32_t> todo{g.root};
  reach[g.root] = 1;
  while (!todo.empty()) {
    const uint32_t r = todo.back();
    todo.pop_back();
    for (uint32_t t : refs[r]) if (!reach[t]) { reach[t] = 1; todo.push_back(t); }
  }
  std::vector<int> color(n, 0);   // iterative DFS for a cycle of left corners: 1 on the path, 2 done
  for (size_t s = 0; s < n; s++) {
    if (!reach[s] || color[s]) continue;
    std::vector<std::pair<uint32_t, size_t>> path{{(uint32_t)s, 0}};
    color[s] = 1;
    while (!path.empty()) {
      auto& top = path.back();
      if (top.second < left[top.first].size()) {
        const uint32_t t = left[top.first][top.second++];
        if (color[t] == 1) throw GrammarError("left recursion through rule '" + g.symbols[t].first + "'", (long)(p - text));
        if (!color[t]) { color[t] = 1; path.push_back({t, 0}); }
      } else {
        color[top.first] = 2;
        path.pop_back();
      }
    }
  }
  return g;
}

// ---------------------------------------------------------------------------------------------------------------------------
// State and acceptance.
struct PartialUtf8 { uint32_t value = 0; int n_remain = 0; };   // n_remain -1: an invalid sequence
using GStack = std::vector<int>;   // element indices, bottom first

struct GrammarState {
  std::vector<GStack> stacks;
  PartialUtf8 partial;
  bool eos_ok() const {
    for (const auto& s : stacks) if (s.empty()) return true;
    return false;
  }
};

// decode_utf8: the piece (up to its first NUL) after the pending partial sequence.  An invalid sequence gives no code points and
// n_remain -1.
inline void decode_utf8(const char* s, size_t n, PartialUtf8 start, std::vector<uint32_t>& cps, PartialUtf8& out) {
  static const int len_of[] = {1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 2, 2, 3, 4};
  cps.clear();
  size_t i = 0;
  const size_t end = std::find(s, s + n, '\0') - s;
  uint32_t v = start.value;
  int rem = start.n_remain;
  while (i < end && rem > 0) {
    const uint8_t b = (uint8_t)s[i];
    if ((b >> 6) != 2) { cps.clear(); out = {0, -1}; return; }
    v = (v << 6) + (b & 0x3F);
    i++;
    rem--;
  }
  if (start.n_remain > 0 && rem == 0) cps.push_back(v);
  while (i < end) {
    const uint8_t b = (uint8_t)s[i];
    rem = len_of[b >> 4] - 1;
    if (rem < 0) { cps.clear(); out = {0, -1}; return; }
    v = b & ((1u << (7 - rem)) - 1);
    i++;
    while (i < end && rem > 0) { v = (v << 6) + ((uint8_t)s[i] & 0x3F); i++; rem--; }
    if (rem == 0) cps.push_back(v);
  }
  out = {v, rem};
}

// llama_grammar_match_char: whether chr satisfies the class at e, and the element after the class
inline bool gmatch_char(const Grammar& g, int e, uint32_t chr, int* after = nullptr) {
  bool found = false;
  const bool pos = g.elems[e].type == G_CHAR;
  do {
    if (g.elems[e + 1].type == G_CHAR_RNG_UPPER) { found = found || (g.elems[e].value <= chr && chr <= g.elems[e + 1].value); e += 2; }
    else { found = found || g.elems[e].value == chr; e += 1; }
  } while (g.elems[e].type == G_CHAR_ALT);
  if (after) *after = e;
  return found == pos;
}

// llama_grammar_match_partial_char: whether some completion of the partial sequence could satisfy the class at e
inline bool gmatch_partial(const Grammar& g, int e, PartialUtf8 pu) {
  const bool pos = g.elems[e].type == G_CHAR;
  if (pu.n_remain < 0 || (pu.n_remain == 1 && pu.value < 2)) return false;
  uint32_t lo = pu.value << (pu.n_remain * 6);
  const uint32_t hi = lo | ((1u << (pu.n_remain * 6)) - 1);
  if (lo == 0) { if (pu.n_remain == 2) lo = 1u << 11; else if (pu.n_remain == 3) lo = 1u << 16; }
  do {
    if (g.elems[e + 1].type == G_CHAR_RNG_UPPER) {
      if (g.elems[e].value <= hi && lo <= g.elems[e + 1].value) return pos;
      e += 2;
    } else {
      if (lo <= g.elems[e].value && g.elems[e].value <= hi) return pos;
      e += 1;
    }
  } while (g.elems[e].type == G_CHAR_ALT);
  return !pos;
}

// llama_grammar_advance_stack: expand rule references on top until every stack ends at a character class (or is empty)
inline void gadvance(const Grammar& g, const GStack& st, std::vector<GStack>& out) {
  if (st.empty()) { out.push_back(st); return; }
  const int e = st.back();
  const GElem x = g.elems[e];
  if (x.type == G_CHAR || x.type == G_CHAR_NOT) { out.push_back(st); return; }
  if (x.type != G_RULE_REF) throw std::logic_error("grammar stack left on a non-terminal element");
  int sub = g.off[x.value];
  for (;;) {
    GStack ns(st.begin(), st.end() - 1);
    if (!g.end_of_seq(e + 1)) ns.push_back(e + 1);
    if (!g.end_of_seq(sub)) ns.push_back(sub);
    gadvance(g, ns, out);
    while (!g.end_of_seq(sub)) sub++;
    if (g.elems[sub].type != G_ALT) break;
    sub++;
  }
}

inline GrammarState grammar_start(const Grammar& g) {
  GrammarState s;
  int e = g.off[g.root];
  for (;;) {
    GStack st;
    if (!g.end_of_seq(e)) st.push_back(e);
    gadvance(g, st, s.stacks);
    while (!g.end_of_seq(e)) e++;
    if (g.elems[e].type != G_ALT) break;
    e++;
  }
  return s;
}

// llama_grammar_accept: the stacks after one code point
inline std::vector<GStack> gaccept_char(const Grammar& g, const std::vector<GStack>& stacks, uint32_t chr) {
  std::vector<GStack> out;
  for (const auto& st : stacks) {
    if (st.empty()) continue;
    int after = 0;
    if (!gmatch_char(g, st.back(), chr, &after)) continue;
    GStack ns(st.begin(), st.end() - 1);
    if (!g.end_of_seq(after)) ns.push_back(after);
    gadvance(g, ns, out);
  }
  return out;
}

// llama_grammar_accept_token, except that what the reference would abort on is refused and leaves the state as it was: EOS when
// no stack is empty, and a piece after which no stack remains.
inline void grammar_accept(const Grammar& g, GrammarState& s, bool is_eos, const std::string& piece) {
  if (is_eos) {
    if (!s.eos_ok()) throw std::invalid_argument("the grammar does not allow the end of the sequence here");
    return;
  }
  std::vector<uint32_t> cps;
  PartialUtf8 pu;
  decode_utf8(piece.data(), piece.size(), s.partial, cps, pu);
  std::vector<GStack> stacks = s.stacks;
  for (uint32_t c : cps) stacks = gaccept_char(g, stacks, c);
  if (stacks.empty()) throw std::invalid_argument("the grammar does not allow this token here");
  s.stacks = std::move(stacks);
  s.partial = pu;
}

// llama_grammar_reject_candidates over candidates {token, code points from `at`, partial}: the candidates every stack rejects
struct GCand { int id; const uint32_t* cp; int n; PartialUtf8 pu; };

std::vector<GCand> greject(const Grammar& g, const std::vector<GStack>& stacks, const std::vector<GCand>& cands);

inline std::vector<GCand> greject_stack(const Grammar& g, const GStack& st, const std::vector<GCand>& cands) {
  std::vector<GCand> rej;
  if (st.empty()) {
    for (const auto& c : cands) if (c.n != 0 || c.pu.n_remain != 0) rej.push_back(c);
    return rej;
  }
  const int top = st.back();
  std::vector<GCand> next;
  for (const auto& c : cands) {
    if (c.n == 0) {
      if (c.pu.n_remain != 0 && !gmatch_partial(g, top, c.pu)) rej.push_back(c);
    } else if (gmatch_char(g, top, c.cp[0])) {
      next.push_back({c.id, c.cp + 1, c.n - 1, c.pu});
    } else {
      rej.push_back(c);
    }
  }
  int after = 0;
  gmatch_char(g, top, 0, &after);
  GStack sa(st.begin(), st.end() - 1);
  if (!g.end_of_seq(after)) sa.push_back(after);
  std::vector<GStack> ns;
  gadvance(g, sa, ns);
  for (const auto& c : greject(g, ns, next)) rej.push_back({c.id, c.cp - 1, c.n + 1, c.pu});
  return rej;
}

inline std::vector<GCand> greject(const Grammar& g, const std::vector<GStack>& stacks, const std::vector<GCand>& cands) {
  if (cands.empty()) return {};
  if (stacks.empty()) throw std::logic_error("grammar state without stacks");
  std::vector<GCand> rej = greject_stack(g, stacks[0], cands);
  for (size_t i = 1; i < stacks.size(); i++) rej = greject_stack(g, stacks[i], rej);
  return rej;
}

// The tokens llama_sample_grammar leaves finite: allowed[t] = 1.  piece(t) gives token t's piece (llama_token_to_str).
template <class Piece>
void grammar_mask(const Grammar& g, const GrammarState& s, int n_vocab, int eos, Piece&& piece, uint8_t* allowed) {
  std::vector<std::vector<uint32_t>> cps(n_vocab);
  std::vector<GCand> cands;
  cands.reserve(n_vocab);
  const bool eos_ok = s.eos_ok();
  for (int t = 0; t < n_vocab; t++) {
    allowed[t] = 0;
    if (t == eos) { allowed[t] = eos_ok; continue; }
    const std::string p = piece(t);
    if (p.empty() || p[0] == 0) continue;
    PartialUtf8 pu;
    decode_utf8(p.data(), p.size(), s.partial, cps[t], pu);
    // the reference's candidate ends at its first code point 0 (the terminator it appends, llama.cpp:3692, 3703): an
    // overlong-encoded NUL ends the piece for the mask; accepting the token still feeds every code point
    cps[t].erase(std::find(cps[t].begin(), cps[t].end(), 0u), cps[t].end());
    allowed[t] = 1;
    cands.push_back({t, cps[t].data(), (int)cps[t].size(), pu});
  }
  for (const auto& c : greject(g, s.stacks, cands)) allowed[c.id] = 0;
}

}  // namespace ctb
