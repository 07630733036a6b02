// Test-only shim over the reference's own grammar_parser::parse (compiled from the reference sources by
// make_golden_grammar.py, never part of the product): flattens the parse_state for ctypes.
#include <cstring>
#include <string>
#include <vector>

#include "grammar-parser.h"

static grammar_parser::parse_state g_state;

extern "C" {
// 0 with the counts, -1 when the parser refused the text (it returns an empty state)
int gp_parse(const char* text, int* n_rules, int* n_elems, int* n_symbols) {
  g_state = grammar_parser::parse(text);
  if (g_state.rules.empty()) return -1;
  int n = 0;
  for (const auto& r : g_state.rules) n += (int)r.size();
  *n_rules = (int)g_state.rules.size();
  *n_elems = n;
  *n_symbols = (int)g_state.symbol_ids.size();
  return 0;
}
// rule r: elems[off[r] .. off[r + 1]) as (type, value) pairs
void gp_rules(int* off, unsigned* elems) {
  int at = 0;
  off[0] = 0;
  for (size_t r = 0; r < g_state.rules.size(); r++) {
    for (const auto& e : g_state.rules[r]) { elems[2 * at] = (unsigned)e.type; elems[2 * at + 1] = e.value; at++; }
    off[r + 1] = at;
  }
}
// the i-th entry of symbol_ids (name order): name length, *id
int gp_symbol(int i, char* name, int cap, unsigned* id) {
  auto it = g_state.symbol_ids.begin();
  std::advance(it, i);
  *id = it->second;
  const int n = (int)it->first.size();
  if (n > cap) return -n;
  memcpy(name, it->first.data(), n);
  return n;
}
}
