// rulec.cpp -- JS RegExp (non-unicode mode, Annex B) -> unit-level Pike program + necessary factors.
// See rulec.h.  Independent of oracle/jsre.c (different data structures and matching model);
// the two only share the language definition, ECMA-262 22.2.
#include "rulec.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <set>

namespace cg {
namespace {

constexpr int INF = 0x7fffffff;

enum NType { T_EMPTY, T_CHAR, T_ANY, T_SET, T_CAT, T_ALT, T_GROUP, T_REPEAT, T_BOL, T_EOL, T_WORDB, T_NWORDB, T_LOOK };

using Ranges = std::vector<std::pair<int, int>>;  // inclusive, over code units 0..0xffff

struct Node {
  int type = T_EMPTY;
  int ch = 0;
  Ranges set;          // T_SET (normalised, positive)
  std::vector<int> kids;
  int min = 0, max = 0;
  bool greedy = true, neg = false, behind = false;
};

struct Fail { int status; std::string msg; };

static void normalise(Ranges& r) {
  std::sort(r.begin(), r.end());
  Ranges o;
  for (auto& p : r) {
    if (!o.empty() && p.first <= o.back().second + 1) o.back().second = std::max(o.back().second, p.second);
    else o.push_back(p);
  }
  r.swap(o);
}
static Ranges negate(const Ranges& r) {
  Ranges o; int lo = 0;
  for (auto& p : r) { if (p.first > lo) o.push_back({lo, p.first - 1}); lo = p.second + 1; }
  if (lo <= 0xffff) o.push_back({lo, 0xffff});
  return o;
}
#include "case_canon.inc"      // kCaseCanon: ECMA-262 Canonicalize for the BMP units >= 0x80 that change (gen_case_table.py)
// units grouped by their canonical form (the form itself included): a class under flag i matches ch iff it holds a member
// with the same canonical form (ECMA-262 22.2.2.9 CharacterSetMatcher)
static const std::vector<std::vector<int>>& canon_groups() {
  static const std::vector<std::vector<int>> groups = [] {
    std::map<int, std::vector<int>> g;
    for (int i = 0; i < kCaseCanonCount; i++) { auto& v = g[kCaseCanon[i][1]]; if (v.empty()) v.push_back(kCaseCanon[i][1]); v.push_back(kCaseCanon[i][0]); }
    std::vector<std::vector<int>> out;
    for (auto& kv : g) out.push_back(kv.second);
    return out;
  }();
  return groups;
}
static bool in_ranges(const Ranges& r, int c) { for (auto& p : r) if (c >= p.first && c <= p.second) return true; return false; }
static void add_case_closure(Ranges& r) {
  Ranges extra;
  for (auto& p : r) {                                    // ASCII letters
    int lo = std::max(p.first, (int)'a'), hi = std::min(p.second, (int)'z');
    if (lo <= hi) extra.push_back({lo - 32, hi - 32});
    lo = std::max(p.first, (int)'A'); hi = std::min(p.second, (int)'Z');
    if (lo <= hi) extra.push_back({lo + 32, hi + 32});
  }
  bool nonascii = false; for (auto& p : r) nonascii |= p.second >= 0x80;
  if (nonascii) for (auto& grp : canon_groups()) {      // everything else: whole groups
    bool any = false; for (int u : grp) if (in_ranges(r, u)) { any = true; break; }
    if (any) for (int u : grp) extra.push_back({u, u});
  }
  r.insert(r.end(), extra.begin(), extra.end());
  normalise(r);
}

static const Ranges kDigit = {{'0', '9'}};
static const Ranges kWord = {{'0', '9'}, {'A', 'Z'}, {'_', '_'}, {'a', 'z'}};
static const Ranges kSpace = {{0x09, 0x0d}, {0x20, 0x20}, {0xa0, 0xa0}, {0x1680, 0x1680}, {0x2000, 0x200a},
                              {0x2028, 0x2029}, {0x202f, 0x202f}, {0x205f, 0x205f}, {0x3000, 0x3000}, {0xfeff, 0xfeff}};

struct Parser {
  std::vector<uint16_t> p;
  size_t i = 0;
  bool icase = false;
  std::vector<Node> nodes;
  int total_groups = 0;
  bool has_named = false;
  bool explicit_nonascii = false;

  int mk(int type) { nodes.emplace_back(); nodes.back().type = type; return (int)nodes.size() - 1; }
  int peek(size_t k = 0) const { return i + k < p.size() ? p[i + k] : -1; }
  [[noreturn]] void syntax(const std::string& m) { throw Fail{RULE_ERR_SYNTAX, m}; }
  [[noreturn]] void unsupported(const std::string& m) { throw Fail{RULE_ERR_UNSUPPORTED, m}; }

  static bool isdig(int c) { return c >= '0' && c <= '9'; }
  static int hexv(int c) {
    if (c >= '0' && c <= '9') return c - '0';
    if (c >= 'a' && c <= 'f') return c - 'a' + 10;
    if (c >= 'A' && c <= 'F') return c - 'A' + 10;
    return -1;
  }

  void prescan() {
    bool in_class = false;
    for (size_t k = 0; k < p.size(); k++) {
      int c = p[k];
      if (c == '\\') { k++; continue; }
      if (in_class) { if (c == ']') in_class = false; continue; }
      if (c == '[') { in_class = true; continue; }
      if (c == '(') {
        if (k + 1 < p.size() && p[k + 1] == '?') {
          if (k + 3 < p.size() && p[k + 2] == '<' && p[k + 3] != '=' && p[k + 3] != '!') { total_groups++; has_named = true; }
        } else total_groups++;
      }
    }
  }

  // body of a character escape after '\' ; returns code unit
  int char_escape(bool in_class) {
    int c = peek();
    if (c < 0) syntax("\\ at end of pattern");
    i++;
    switch (c) {
      case 't': return 0x09; case 'n': return 0x0a; case 'v': return 0x0b; case 'f': return 0x0c; case 'r': return 0x0d;
      case 'b': if (in_class) return 0x08; break;
      case '0': if (!isdig(peek())) return 0; break;
      case 'c': {
        int l = peek();
        if ((l >= 'a' && l <= 'z') || (l >= 'A' && l <= 'Z')) { i++; return l % 32; }
        if (in_class && (isdig(l) || l == '_')) { i++; return l % 32; }
        i--; return '\\';
      }
      case 'x': { int a = hexv(peek()), b = hexv(peek(1)); if (a >= 0 && b >= 0) { i += 2; return a * 16 + b; } return 'x'; }
      case 'u': {
        int v = 0; bool ok = true;
        for (int k = 0; k < 4; k++) { int h = hexv(peek(k)); if (h < 0) { ok = false; break; } v = v * 16 + h; }
        if (ok) { i += 4; return v; }
        return 'u';
      }
      case 'k': if (has_named) unsupported("named backreference"); break;
    }
    if (c >= '0' && c <= '7') {
      int v = c - '0'; int d = peek();
      if (d >= '0' && d <= '7') { v = v * 8 + (d - '0'); i++; d = peek(); if (c <= '3' && d >= '0' && d <= '7') { v = v * 8 + (d - '0'); i++; } }
      return v;
    }
    return c;
  }

  static const Ranges* class_escape(int c, bool* inv) {
    *inv = (c == 'D' || c == 'W' || c == 'S');
    switch (c) { case 'd': case 'D': return &kDigit; case 'w': case 'W': return &kWord; case 's': case 'S': return &kSpace; }
    return nullptr;
  }
  static void add_set(Ranges& r, const Ranges& s, bool inv) {
    if (!inv) { r.insert(r.end(), s.begin(), s.end()); return; }
    Ranges n = negate(s); r.insert(r.end(), n.begin(), n.end());
  }

  int finish_set(Ranges r, bool neg) {
    normalise(r);
    if (icase) add_case_closure(r);
    if (neg) r = negate(r);
    int n = mk(T_SET); nodes[n].set = r; return n;
  }

  int parse_class() {
    bool neg = false; Ranges r;
    if (peek() == '^') { neg = true; i++; }
    for (;;) {
      int c = peek();
      if (c < 0) syntax("unterminated character class");
      if (c == ']') { i++; break; }
      i++;
      int lo = -1; bool lo_set = false;
      if (c == '\\') {
        bool inv; const Ranges* s = class_escape(peek(), &inv);
        if (s) { i++; add_set(r, *s, inv); lo_set = true; } else lo = char_escape(true);
      } else lo = c;
      if (peek() == '-' && peek(1) != ']' && peek(1) >= 0) {
        i++;
        int c2 = peek(); i++;
        int hi = -1;
        if (c2 == '\\') {
          bool inv; const Ranges* s = class_escape(peek(), &inv);
          if (s) { i++; if (!lo_set) { r.push_back({lo, lo}); if (lo >= 128) explicit_nonascii = true; } r.push_back({'-', '-'}); add_set(r, *s, inv); continue; }
          hi = char_escape(true);
        } else hi = c2;
        if (lo_set) { r.push_back({'-', '-'}); r.push_back({hi, hi}); if (hi >= 128) explicit_nonascii = true; continue; }
        if (hi < lo) syntax("range out of order in character class");
        r.push_back({lo, hi});
        if (hi >= 128) explicit_nonascii = true;
        continue;
      }
      if (!lo_set) { r.push_back({lo, lo}); if (lo >= 128) explicit_nonascii = true; }
    }
    return finish_set(r, neg);
  }

  bool braces(int* mn, int* mx) {
    size_t j = i;
    if (j >= p.size() || p[j] != '{') return false;
    j++;
    if (j >= p.size() || !isdig(p[j])) return false;
    long a = 0; while (j < p.size() && isdig(p[j])) { a = std::min(a * 10 + (p[j] - '0'), (long)INF); j++; }
    long b = a;
    if (j < p.size() && p[j] == ',') {
      j++;
      if (j < p.size() && isdig(p[j])) { b = 0; while (j < p.size() && isdig(p[j])) { b = std::min(b * 10 + (p[j] - '0'), (long)INF); j++; } }
      else b = INF;
    }
    if (j >= p.size() || p[j] != '}') return false;
    i = j + 1; *mn = (int)a; *mx = (int)b; return true;
  }

  int mkchar(int c) {
    if (c >= 128) explicit_nonascii = true;
    if (icase && ((c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || c >= 0x80)) return finish_set({{c, c}}, false);
    int n = mk(T_CHAR); nodes[n].ch = c; return n;
  }

  int atom_escape(bool* is_assert) {
    int c = peek();
    bool inv; const Ranges* s = class_escape(c, &inv);
    if (s) { i++; Ranges r; add_set(r, *s, inv); return finish_set(r, false); }
    if (c == 'b') { i++; *is_assert = true; return mk(T_WORDB); }
    if (c == 'B') { i++; *is_assert = true; return mk(T_NWORDB); }
    if (c >= '1' && c <= '9') {
      size_t j = i; long v = 0;
      while (j < p.size() && isdig(p[j])) { v = std::min(v * 10 + (p[j] - '0'), 100000L); j++; }
      if (v <= total_groups) unsupported("backreference");
      if (c >= '8') { i++; return mkchar(c); }
    }
    return mkchar(char_escape(false));
  }

  int parse_disjunction();

  int parse_term(bool* is_assert) {
    *is_assert = false;
    int c = peek(); i++;
    switch (c) {
      case '^': *is_assert = true; return mk(T_BOL);
      case '$': *is_assert = true; return mk(T_EOL);
      case '.': return mk(T_ANY);
      case '[': return parse_class();
      case '\\': return atom_escape(is_assert);
      case '(': {
        int atom;
        if (peek() == '?') {
          int d = peek(1);
          if (d == ':') { i += 2; atom = mk(T_GROUP); int k = parse_disjunction(); nodes[atom].kids.push_back(k); }
          else if (d == '=' || d == '!') {
            i += 2; atom = mk(T_LOOK); nodes[atom].neg = (d == '!'); nodes[atom].behind = false;
            int k = parse_disjunction(); nodes[atom].kids.push_back(k);
          } else if (d == '<' && (peek(2) == '=' || peek(2) == '!')) {
            bool neg = peek(2) == '!'; i += 3; atom = mk(T_LOOK); nodes[atom].neg = neg; nodes[atom].behind = true;
            int k = parse_disjunction(); nodes[atom].kids.push_back(k);
            *is_assert = true;
          } else if (d == '<') {
            i += 2; while (peek() >= 0 && peek() != '>') i++;
            if (peek() != '>') syntax("invalid capture group name");
            i++; atom = mk(T_GROUP); int k = parse_disjunction(); nodes[atom].kids.push_back(k);
          } else syntax("invalid group");
        } else { atom = mk(T_GROUP); int k = parse_disjunction(); nodes[atom].kids.push_back(k); }
        if (peek() != ')') syntax("unterminated group");
        i++;
        return atom;
      }
      case '*': case '+': case '?': syntax("nothing to repeat");
      case '{': { i--; int a, b; size_t sv = i; if (braces(&a, &b)) { i = sv; syntax("nothing to repeat"); } i++; return mkchar('{'); }
      default: return mkchar(c);
    }
  }

  int parse_alternative() {
    int seq = mk(T_CAT);
    for (;;) {
      int c = peek();
      if (c < 0 || c == '|' || c == ')') break;
      bool is_assert = false;
      int t = parse_term(&is_assert);
      if (!is_assert) {
        int mn = -1, mx = -1; int q = peek();
        if (q == '*') { mn = 0; mx = INF; i++; } else if (q == '+') { mn = 1; mx = INF; i++; }
        else if (q == '?') { mn = 0; mx = 1; i++; } else if (q == '{') { if (!braces(&mn, &mx)) mn = -1; }
        if (mn >= 0) {
          if (mx < mn) syntax("numbers out of order in {} quantifier");
          if (nodes[t].type == T_LOOK) unsupported("quantified lookahead");
          int r = mk(T_REPEAT); nodes[r].min = mn; nodes[r].max = mx; nodes[r].greedy = true;
          if (peek() == '?') { nodes[r].greedy = false; i++; }
          nodes[r].kids.push_back(t); t = r;
          int q2 = peek();
          if (q2 == '*' || q2 == '+' || q2 == '?') syntax("nothing to repeat");
          int a, b; size_t sv = i; if (q2 == '{' && braces(&a, &b)) { i = sv; syntax("nothing to repeat"); }
        }
      }
      nodes[seq].kids.push_back(t);
    }
    return seq;
  }
};

int Parser::parse_disjunction() {
  int first = parse_alternative();
  if (peek() != '|') return first;
  int alt = mk(T_ALT); nodes[alt].kids.push_back(first);
  while (peek() == '|') { i++; int k = parse_alternative(); nodes[alt].kids.push_back(k); }
  return alt;
}

// ------------------------------------------------------------------ analysis + emission

struct Compiler {
  Parser& ps;
  CompiledRule& out;
  explicit Compiler(Parser& p, CompiledRule& o) : ps(p), out(o) {}
  const Node& N(int n) const { return ps.nodes[n]; }

  bool nullable(int n) const {
    const Node& nd = N(n);
    switch (nd.type) {
      case T_CHAR: case T_ANY: case T_SET: return false;
      case T_CAT: for (int k : nd.kids) if (!nullable(k)) return false; return true;
      case T_ALT: for (int k : nd.kids) if (nullable(k)) return true; return false;
      case T_GROUP: return nullable(nd.kids[0]);
      case T_REPEAT: return nd.min == 0 || nullable(nd.kids[0]);
      default: return true;
    }
  }

  void check_supported(int n) {
    const Node& nd = N(n);
    if (nd.type == T_LOOK) {
      int k = nd.kids[0];
      for (;;) {
        const Node& kn = N(k);
        if ((kn.type == T_GROUP || kn.type == T_CAT || kn.type == T_ALT) && kn.kids.size() == 1) { k = kn.kids[0]; continue; }
        break;
      }
      int t = N(k).type;
      if (t != T_CHAR && t != T_SET && t != T_ANY) throw Fail{RULE_ERR_UNSUPPORTED, "lookaround over more than one character"};
    }
    for (int k : nd.kids) check_supported(k);
  }

  static Ranges any_set() { return negate({{0x0a, 0x0a}, {0x0d, 0x0d}, {0x2028, 0x2029}}); }
  Ranges unit_ranges(int n) const {
    const Node& nd = N(n);
    if (nd.type == T_CHAR) return {{nd.ch, nd.ch}};
    if (nd.type == T_ANY) return any_set();
    return nd.set;
  }

  int set_id(const Ranges& r) {
    UnitSet s; memset(s.ascii, 0, sizeof s.ascii);
    for (auto& p : r) {
      for (int c = p.first; c <= std::min(p.second, 127); c++) s.ascii[c >> 5] |= 1u << (c & 31);
      if (p.second >= 128) { s.ranges.push_back((uint16_t)std::max(p.first, 128)); s.ranges.push_back((uint16_t)p.second); }
    }
    for (size_t k = 0; k < out.sets.size(); k++) if (out.sets[k] == s) return (int)k;
    out.sets.push_back(s);
    return (int)out.sets.size() - 1;
  }

  void emit(uint32_t op, uint32_t arg = 0) {
    if ((int)out.prog.size() >= kMaxProgLen) throw Fail{RULE_ERR_TOO_LARGE, "pattern expands to more than 1024 matcher instructions"};
    out.prog.push_back(op | (arg << 8));
  }
  void patch(size_t at, uint32_t arg) { out.prog[at] = (out.prog[at] & 0xff) | (arg << 8); }

  void gen(int n) {
    const Node& nd = N(n);
    switch (nd.type) {
      case T_EMPTY: return;
      case T_CHAR: emit(OP_CHAR, (uint32_t)nd.ch); return;
      case T_ANY: emit(OP_ANY); return;
      case T_SET: {
        if (nd.set.size() == 1 && nd.set[0].first == nd.set[0].second) { emit(OP_CHAR, (uint32_t)nd.set[0].first); return; }
        emit(OP_SET, (uint32_t)set_id(nd.set)); return;
      }
      case T_CAT: for (int k : nd.kids) gen(k); return;
      case T_GROUP: gen(nd.kids[0]); return;
      case T_ALT: {
        std::vector<size_t> jumps;
        for (size_t a = 0; a < nd.kids.size(); a++) {
          if (a + 1 < nd.kids.size()) {
            size_t sp = out.prog.size(); emit(OP_SPLIT_NEXT, 0);
            gen(nd.kids[a]);
            jumps.push_back(out.prog.size()); emit(OP_JMP, 0);
            patch(sp, (uint32_t)out.prog.size());
          } else gen(nd.kids[a]);
        }
        for (size_t j : jumps) patch(j, (uint32_t)out.prog.size());
        return;
      }
      case T_REPEAT: {
        int body = nd.kids[0];
        // (a body that emits nothing -- `(?:){2000000000}` -- is never stopped by the program-length limit: once is enough)
        for (int c = 0; c < nd.min; c++) { const size_t before = out.prog.size(); gen(body); if (out.prog.size() == before) break; }
        if (nd.max == INF) {
          size_t L = out.prog.size();
          emit(nd.greedy ? OP_SPLIT_NEXT : OP_SPLIT_JUMP, 0);
          gen(body);
          emit(OP_JMP_BACK, (uint32_t)L);
          patch(L, (uint32_t)out.prog.size());
        } else {
          // optional iterations: RepeatMatcher's empty check (22.2.2.3.1 step 2.b) rejects an
          // iteration that consumed nothing; EMPTYCHK tests the visited mark of this iteration's SPLIT.
          std::vector<size_t> splits; bool nb = nullable(body);
          for (int c = nd.min; c < nd.max; c++) {
            if (out.prog.size() > (size_t)kMaxProgLen) break;                   // (emit() reports the overflow)
            splits.push_back(out.prog.size()); emit(nd.greedy ? OP_SPLIT_NEXT : OP_SPLIT_JUMP, 0);
            gen(body);
            if (nb) emit(OP_EMPTYCHK, (uint32_t)splits.back());
          }
          for (size_t s : splits) patch(s, (uint32_t)out.prog.size());
        }
        return;
      }
      case T_BOL: emit(OP_BOL); return;
      case T_EOL: emit(OP_EOL); return;
      case T_WORDB: emit(OP_WORDB); return;
      case T_NWORDB: emit(OP_NWORDB); return;
      case T_LOOK: {
        int k = nd.kids[0];
        for (;;) { const Node& kn = N(k); if ((kn.type == T_GROUP || kn.type == T_CAT || kn.type == T_ALT) && kn.kids.size() == 1) { k = kn.kids[0]; continue; } break; }
        int sid = set_id(unit_ranges(k));
        uint32_t op = nd.behind ? (nd.neg ? OP_NLOOKBEHIND : OP_LOOKBEHIND) : (nd.neg ? OP_NLOOKAHEAD : OP_LOOKAHEAD);
        emit(op, (uint32_t)sid); return;
      }
    }
  }

  // FIRST set (units) of a node
  void first(int n, Ranges& acc) const {
    const Node& nd = N(n);
    switch (nd.type) {
      case T_CHAR: case T_ANY: case T_SET: { Ranges r = unit_ranges(n); acc.insert(acc.end(), r.begin(), r.end()); return; }
      case T_CAT: for (int k : nd.kids) { first(k, acc); if (!nullable(k)) return; } return;
      case T_ALT: for (int k : nd.kids) first(k, acc); return;
      case T_GROUP: case T_REPEAT: first(nd.kids[0], acc); return;
      default: return;
    }
  }

  // ---------------------------------------------------------------- necessary factors
  struct Info {
    bool has_exact = false;             // language(node) subset of `exact` (as whole strings)
    std::vector<FactorSeq> exact;
    bool is_exact_tight = false;        // `exact` IS the language (no over-approximation, no assertions)
    bool has_factors = false;           // every match contains one of `factors` as a substring
    std::vector<FactorSeq> factors;
    int fpre = 0;                       // max units of the node's match that can precede that factor occurrence (kPreInf = unbounded)
    ByteSet fpre_alpha;                 // bytes that part of the match before the factor can consist of (over-approximation)
  };
  // every byte the sub-pattern can consume
  ByteSet alpha_of(int n) const {
    const Node& nd = N(n); ByteSet a;
    if (nd.type == T_CHAR || nd.type == T_ANY || nd.type == T_SET) {
      Ranges r = unit_ranges(n);
      for (auto& p : r) { for (int b = p.first; b <= std::min(p.second, 127); b++) a.set(b); if (p.second >= 128) for (int b = 128; b < 256; b++) a.set(b); }
      return a;
    }
    if (nd.type == T_LOOK) return a;
    for (int k : nd.kids) { ByteSet s = alpha_of(k); for (int i = 0; i < 4; i++) a.w[i] |= s.w[i]; }
    return a;
  }
  static void or_into(ByteSet& a, const ByteSet& b) { for (int i = 0; i < 4; i++) a.w[i] |= b.w[i]; }
  static constexpr int kPreInf = 1 << 20;
  int maxlen(int n) const {
    const Node& nd = N(n); long v = 0;
    switch (nd.type) {
      case T_CHAR: case T_ANY: case T_SET: return 1;
      case T_CAT: for (int k : nd.kids) { v += maxlen(k); if (v >= kPreInf) return kPreInf; } return (int)v;
      case T_ALT: for (int k : nd.kids) v = std::max<long>(v, maxlen(k)); return (int)v;
      case T_GROUP: return maxlen(nd.kids[0]);
      case T_REPEAT: { if (nd.max == INF) return maxlen(nd.kids[0]) ? kPreInf : 0; long m = (long)nd.max * maxlen(nd.kids[0]); return m >= kPreInf ? kPreInf : (int)m; }
      default: return 0;
    }
  }
  static constexpr size_t kMaxSeqs = 24;
  static constexpr size_t kMaxRunLen = 16;

  static double byte_weight(int b) {
    // coarse frequency model of chat-like UTF-8 text, used only to rank factor candidates
    if (b == ' ') return 0.15;
    if (b >= 'a' && b <= 'z') { static const double f[26] = {.065,.012,.022,.034,.10,.018,.016,.049,.056,.001,.006,.032,.019,.054,.060,.015,.001,.048,.051,.072,.022,.008,.019,.001,.016,.001}; return f[b - 'a']; }
    if (b >= 'A' && b <= 'Z') return 0.002;
    if (b >= '0' && b <= '9') return 0.004;
    if (b == '.' || b == ',') return 0.01;
    if (b >= 0x21 && b <= 0x7e) return 0.0015;
    if (b == '\n') return 0.003;
    if (b >= 0x80) return 0.0004;
    return 0.0001;
  }
  static double seq_prob(const FactorSeq& s) {
    double p = 1.0;
    for (auto& bs : s) { double q = 0; for (int b = 0; b < 256; b++) if (bs.has(b)) q += byte_weight(b); p *= std::min(q, 1.0); }
    return p;
  }
  static double score(const std::vector<FactorSeq>& f) {
    double s = 0; for (auto& q : f) { if (q.empty()) return 1.0; s += seq_prob(q); } return std::min(s, 1.0);
  }

  // byte-level view of one unit node.  ASCII-only sets are one exact byte set; a single non-ASCII
  // literal is its UTF-8 bytes; any other set with members >= 0x80 is over-approximated by the three
  // byte shapes one decoded unit can have (1 byte; 2 bytes incl. half an astral pair or a truncated
  // sequence; 3 bytes) -- sound for ill-formed input too, since every U+FFFD the decoder emits
  // covers 1-3 bytes of exactly these shapes.  U+FFFD itself therefore takes the three shapes even
  // as a single literal: EF BF BD is only one of the byte strings it decodes from.  *tight is
  // cleared when the view over-approximates.
  bool unit_bytes(int n, std::vector<FactorSeq>* seqs, bool* tight) const {
    Ranges r = unit_ranges(n);
    *tight = true;
    bool ascii_only = true; for (auto& p : r) if (p.second >= 128) ascii_only = false;
    ByteSet lo; for (auto& p : r) for (int c = p.first; c <= std::min(p.second, 127); c++) lo.set(c);
    if (ascii_only) { if (lo.empty()) return false; seqs->push_back({lo}); return true; }
    if (r.size() == 1 && r[0].first == r[0].second) {      // single non-ASCII literal: its UTF-8 bytes
      int c = r[0].first;
      if (!(c >= 0xd800 && c <= 0xdfff) && c != 0xfffd) {
        FactorSeq s; ByteSet b0, b1, b2;
        if (c < 0x800) { b0.set(0xc0 | (c >> 6)); b1.set(0x80 | (c & 0x3f)); s = {b0, b1}; }
        else { b0.set(0xe0 | (c >> 12)); b1.set(0x80 | ((c >> 6) & 0x3f)); b2.set(0x80 | (c & 0x3f)); s = {b0, b1, b2}; }
        seqs->push_back(s); return true;
      }
    }
    *tight = false;
    ByteSet one = lo, hi, cont, lead3;
    for (int b = 0x80; b < 0x100; b++) { one.set(b); hi.set(b); }
    for (int b = 0x80; b < 0xc0; b++) cont.set(b);
    for (int b = 0xe0; b <= 0xf4; b++) lead3.set(b);
    seqs->push_back({one}); seqs->push_back({hi, cont}); seqs->push_back({lead3, cont, cont});
    return true;
  }

  static void consider(std::vector<FactorSeq>& best, bool& have, int& best_pre, ByteSet& best_alpha, const std::vector<FactorSeq>& cand, int cand_pre,
                       const ByteSet& cand_alpha) {
    if (cand.empty()) return;
    for (auto& s : cand) if (s.empty()) return;
    if (!have || score(cand) < score(best)) { best = cand; have = true; best_pre = std::min(cand_pre, kPreInf); best_alpha = cand_alpha; }
  }

  Info analyse(int n) const {
    const Node& nd = N(n);
    Info I;
    switch (nd.type) {
      case T_CHAR: case T_ANY: case T_SET: {
        std::vector<FactorSeq> s; bool tight = true;
        if (unit_bytes(n, &s, &tight)) { I.has_exact = true; I.exact = s; I.is_exact_tight = tight; I.has_factors = true; I.factors = s; }
        return I;
      }
      case T_EMPTY: I.has_exact = true; I.exact = {FactorSeq{}}; I.is_exact_tight = true; return I;
      case T_BOL: case T_EOL: case T_WORDB: case T_NWORDB: case T_LOOK:
        I.has_exact = true; I.exact = {FactorSeq{}}; I.is_exact_tight = false; return I;
      case T_GROUP: return analyse(nd.kids[0]);
      case T_ALT: {
        bool all_exact = true, all_fact = true, tight = true; std::vector<FactorSeq> ex, fa;
        for (int k : nd.kids) {
          Info c = analyse(k);
          if (c.has_exact) ex.insert(ex.end(), c.exact.begin(), c.exact.end()); else all_exact = false;
          tight = tight && c.is_exact_tight;
          if (c.has_factors) { fa.insert(fa.end(), c.factors.begin(), c.factors.end()); I.fpre = std::max(I.fpre, c.fpre); or_into(I.fpre_alpha, c.fpre_alpha); } else all_fact = false;
        }
        if (all_exact && ex.size() <= kMaxSeqs) { I.has_exact = true; I.exact = ex; I.is_exact_tight = tight; }
        if (all_fact && fa.size() <= 4 * kMaxSeqs) { I.has_factors = true; I.factors = fa; }
        return I;
      }
      case T_REPEAT: {
        // view X{m,n} as X^m followed by an optional tail (which gives no information)
        Info b = analyse(nd.kids[0]);
        if (nd.min == 0) { if (nd.max == 0) { I.has_exact = true; I.exact = {FactorSeq{}}; I.is_exact_tight = true; } return I; }
        std::vector<FactorSeq> run; bool have = false;
        if (b.has_exact) {
          run = {FactorSeq{}};
          int copies = std::min(nd.min, (int)kMaxRunLen);
          bool ok = true;
          for (int c = 0; c < copies && ok; c++) {
            std::vector<FactorSeq> nx;
            for (auto& a : run) for (auto& e : b.exact) { FactorSeq s = a; s.insert(s.end(), e.begin(), e.end()); if (s.size() > kMaxRunLen) { ok = false; break; } nx.push_back(s); }
            if (!ok || nx.size() > kMaxSeqs) { ok = false; break; }
            run.swap(nx);
          }
          if (!run.empty() && !run[0].empty()) {
            have = true;
            if (ok && nd.min == nd.max && copies == nd.min) { I.has_exact = true; I.exact = run; I.is_exact_tight = b.is_exact_tight; }
          }
        }
        std::vector<FactorSeq> best; bool hb = false; int bpre = 0; ByteSet balpha;
        if (have) consider(best, hb, bpre, balpha, run, 0, ByteSet());
        if (b.has_factors) {
          int ml = maxlen(nd.kids[0]);
          long before = nd.max == INF ? (ml ? kPreInf : 0) : (long)(nd.max - 1) * ml;
          ByteSet al = b.fpre_alpha; if (nd.max != 1) or_into(al, alpha_of(nd.kids[0]));     // earlier iterations of the body
          consider(best, hb, bpre, balpha, b.factors, (int)std::min<long>(before + b.fpre, kPreInf), al);
        }
        if (hb) { I.has_factors = true; I.factors = best; I.fpre = bpre; I.fpre_alpha = balpha; }
        return I;
      }
      case T_CAT: {
        std::vector<FactorSeq> run = {FactorSeq{}}; bool run_tight = true;
        std::vector<FactorSeq> best; bool hb = false; int bpre = 0; ByteSet balpha;
        bool all_exact = true, tight = true;
        long pos = 0; int run_pre = 0;      // pos: max units consumed by the children before the current one
        ByteSet alpha_before, run_alpha;    // bytes the children before the current one / before the run can consume
        auto run_is_empty = [&]() { return run.size() == 1 && run[0].empty(); };
        auto close_run = [&]() { bool nonempty = false; for (auto& s : run) if (!s.empty()) nonempty = true; bool allne = true; for (auto& s : run) if (s.empty()) allne = false; if (nonempty && allne) consider(best, hb, bpre, balpha, run, run_pre, run_alpha); run = {FactorSeq{}}; };
        for (int k : nd.kids) {
          Info c = analyse(k);
          const int pre_k = (int)std::min<long>(pos, kPreInf);
          pos = std::min<long>(pos + maxlen(k), kPreInf);
          const ByteSet alpha_k = alpha_before;
          or_into(alpha_before, alpha_of(k));
          if (c.has_factors) { ByteSet al = alpha_k; or_into(al, c.fpre_alpha); consider(best, hb, bpre, balpha, c.factors, (int)std::min<long>((long)pre_k + c.fpre, kPreInf), al); }
          if (run_is_empty()) { run_pre = pre_k; run_alpha = alpha_k; }
          // a REPEAT with min>=1 contributes its required prefix to the run and then breaks it
          const Node& kn = N(k);
          bool breaks_after = false;
          std::vector<FactorSeq> piece; bool has_piece = false;
          if (c.has_exact) { piece = c.exact; has_piece = true; tight = tight && c.is_exact_tight; }
          else {
            all_exact = false;
            int kk = k; while (N(kk).type == T_GROUP) kk = N(kk).kids[0];
            if (N(kk).type == T_REPEAT && N(kk).min >= 1) {
              Info b = analyse(N(kk).kids[0]);
              if (b.has_exact) {
                piece = {FactorSeq{}}; has_piece = true; breaks_after = true;
                int copies = std::min(N(kk).min, (int)kMaxRunLen);
                for (int q = 0; q < copies && has_piece; q++) {
                  std::vector<FactorSeq> nx; bool full = false;
                  for (auto& a : piece) for (auto& e : b.exact) { FactorSeq s = a; s.insert(s.end(), e.begin(), e.end()); if (s.size() >= kMaxRunLen) { s.resize(kMaxRunLen); full = true; } nx.push_back(s); }
                  if (nx.size() > kMaxSeqs) break;
                  piece.swap(nx);
                  if (full) break;
                }
              }
            }
            (void)kn;
          }
          if (!has_piece) { close_run(); run_tight = false; continue; }
          // extend the run by the cross product; a piece that would overflow the element limit is
          // cut (a prefix of a necessary factor is still necessary) and the run is closed there
          std::vector<FactorSeq> nx; bool cut = false;
          for (auto& a : run) for (auto& e : piece) {
            FactorSeq s = a; s.insert(s.end(), e.begin(), e.end());
            if (s.size() > kMaxRunLen) { s.resize(kMaxRunLen); cut = true; }
            nx.push_back(s);
          }
          if (nx.size() > kMaxSeqs) { all_exact = false; close_run(); run = piece; run_pre = pre_k; run_alpha = alpha_k; if (run.size() > kMaxSeqs) run = {FactorSeq{}}; for (auto& s : run) if (s.size() > kMaxRunLen) { s.resize(kMaxRunLen); cut = true; } }
          else run.swap(nx);
          if (cut) { all_exact = false; close_run(); }
          if (breaks_after) { all_exact = false; close_run(); }
        }
        if (all_exact) { I.has_exact = true; I.exact = run; I.is_exact_tight = tight && run_tight; }
        close_run();
        if (hb) { I.has_factors = true; I.factors = best; I.fpre = bpre; I.fpre_alpha = balpha; }
        if (I.has_exact && !I.has_factors) { bool allne = true; for (auto& s : I.exact) if (s.empty()) allne = false; if (allne && !I.exact.empty()) { I.has_factors = true; I.factors = I.exact; I.fpre = 0; } }
        return I;
      }
    }
    return I;
  }
};

static std::vector<uint16_t> utf8_to_units(const char* s, size_t n) {
  std::vector<uint16_t> u; size_t i = 0;
  auto* p = reinterpret_cast<const unsigned char*>(s);
  while (i < n) {
    uint32_t c = p[i];
    if (c < 0x80) { u.push_back((uint16_t)c); i++; continue; }
    int need = 0; uint32_t cp = 0, lo = 0x80, hi = 0xbf;
    if (c >= 0xc2 && c <= 0xdf) { need = 1; cp = c & 0x1f; }
    else if (c >= 0xe0 && c <= 0xef) { need = 2; cp = c & 0x0f; if (c == 0xe0) lo = 0xa0; if (c == 0xed) hi = 0x9f; }
    else if (c >= 0xf0 && c <= 0xf4) { need = 3; cp = c & 0x07; if (c == 0xf0) lo = 0x90; if (c == 0xf4) hi = 0x8f; }
    else { u.push_back(0xfffd); i++; continue; }
    size_t j = i + 1; bool ok = true;
    for (int t = 0; t < need; t++, j++) { if (j >= n || p[j] < lo || p[j] > hi) { ok = false; break; } cp = (cp << 6) | (p[j] & 0x3f); lo = 0x80; hi = 0xbf; }
    if (!ok) { u.push_back(0xfffd); i = j > i + 1 ? j : i + 1; continue; }
    i = j;
    if (cp >= 0x10000) { cp -= 0x10000; u.push_back((uint16_t)(0xd800 + (cp >> 10))); u.push_back((uint16_t)(0xdc00 + (cp & 0x3ff))); }
    else u.push_back((uint16_t)cp);
  }
  return u;
}

}  // namespace

// Worst-case depth of the VM's closure stack (pike_vm.h, VMS::add) for this program: the closure walk is replayed from
// every pc a closure can start at, with every zero-width assertion passing and fresh marks (a real run only ever cuts
// paths: assertions fail, marks of earlier threads are DONE).  The device stack holds kVmStackLimit entries; a rule that
// could overflow it is rejected at compile time instead of failing every batch it meets at scan time.
static int closure_stack_bound(const std::vector<uint32_t>& prog) {
  const size_t n = prog.size();
  std::vector<char> starts(n, 0);
  if (n) starts[0] = 1;
  for (size_t pc = 0; pc + 1 < n; pc++) { uint32_t op = prog[pc] & 0xff; if (op == OP_CHAR || op == OP_SET || op == OP_ANY) starts[pc + 1] = 1; }
  int worst = 0;
  std::vector<uint8_t> mark(n); std::vector<uint32_t> stk;
  for (size_t s0 = 0; s0 < n; s0++) {
    if (!starts[s0]) continue;
    std::fill(mark.begin(), mark.end(), 0);           // 0 = untouched, 1 = in progress, 2 = done
    stk.clear(); stk.push_back((uint32_t)s0);
    while (!stk.empty()) {
      worst = std::max<int>(worst, (int)stk.size());
      uint32_t x = stk.back(); stk.pop_back();
      if (x & 0x80000000u) { mark[x & 0x7fffffffu] = 2; continue; }
      uint32_t pc = x;
      for (;;) {
        if (pc >= n) break;
        const uint32_t op = prog[pc] & 0xff, arg = prog[pc] >> 8; bool go = false;
        switch (op) {
          case OP_SPLIT_NEXT: case OP_SPLIT_JUMP:
            if (mark[pc] == 2) break;
            mark[pc] = 1;
            stk.push_back(0x80000000u | pc); stk.push_back(op == OP_SPLIT_NEXT ? arg : pc + 1);
            worst = std::max<int>(worst, (int)stk.size());
            if (worst > 4 * kVmStackLimit) return worst;
            pc = op == OP_SPLIT_NEXT ? pc + 1 : arg; go = true; break;
          case OP_JMP: pc = arg; go = true; break;
          case OP_JMP_BACK: if (mark[arg] != 1) { pc = arg; go = true; } break;
          case OP_EMPTYCHK: if (mark[arg] != 1) { pc++; go = true; } break;
          case OP_BOL: case OP_EOL: case OP_WORDB: case OP_NWORDB: case OP_LOOKAHEAD: case OP_NLOOKAHEAD: case OP_LOOKBEHIND: case OP_NLOOKBEHIND:
            pc++; go = true; break;
          case OP_MATCH: break;
          default: mark[pc] = 2; break;        // consuming instruction: the thread is queued
        }
        if (!go) break;
      }
    }
  }
  return worst;
}

CompiledRule compile_rule(const char* src, size_t len, uint32_t flags) {
  CompiledRule out;
  Parser ps;
  ps.p = utf8_to_units(src, len);
  ps.icase = flags & 1;
  try {
    ps.prescan();
    int root = ps.parse_disjunction();
    if (ps.i < ps.p.size()) throw Fail{RULE_ERR_SYNTAX, ps.p[ps.i] == ')' ? "unmatched ')'" : "unexpected character"};
    Compiler c(ps, out);
    c.check_supported(root);
    c.gen(root);
    c.emit(OP_MATCH);
    if (closure_stack_bound(out.prog) > kVmStackLimit) throw Fail{RULE_ERR_TOO_LARGE, "pattern nests / alternates too deeply for the matcher's closure stack"};
    out.nullable = c.nullable(root);
    if (out.nullable) { for (int k = 0; k < 4; k++) out.first_bytes.w[k] = ~0ull; }
    else {
      Ranges f; c.first(root, f); normalise(f);
      for (auto& p : f) { for (int b = p.first; b <= std::min(p.second, 127); b++) out.first_bytes.set(b); if (p.second >= 128) for (int b = 128; b < 256; b++) out.first_bytes.set(b); }
    }
    // alphabet: union of everything the pattern can consume (a match never contains other bytes)
    for (const Node& nd : ps.nodes) {
      if (nd.type != T_CHAR && nd.type != T_ANY && nd.type != T_SET) continue;
      Ranges r = nd.type == T_CHAR ? Ranges{{nd.ch, nd.ch}} : nd.type == T_ANY ? Compiler::any_set() : nd.set;
      for (auto& p : r) { for (int b = p.first; b <= std::min(p.second, 127); b++) out.alphabet.set(b); if (p.second >= 128) for (int b = 128; b < 256; b++) out.alphabet.set(b); }
    }
    if (!out.nullable) {
      Compiler::Info I = c.analyse(root);
      if (I.has_factors) {
        bool ok = !I.factors.empty(); for (auto& s : I.factors) if (s.empty()) ok = false;
        if (ok) {
          out.factors = I.factors;
          out.factor_pre = I.fpre;
          out.factor_pre_alpha = I.fpre_alpha;
          out.factors_exact = I.has_exact && I.is_exact_tight && I.exact == I.factors;
        }
      }
    }
  } catch (const Fail& f) {
    out = CompiledRule();
    out.status = f.status; out.error = f.msg;
  }
  return out;
}

// ------------------------------------------------------------------ prefilter (gram filter, see rulec.h)

namespace {
struct GramChoice { int off = 0; double count = 1e300, prob = 2; int inside = 0; bool ok = false; };
}  // namespace

bool build_prefilter(const std::vector<CompiledRule>& rules, const PrefilterOptions& opt, Prefilter* pf, std::string* err) {
  Prefilter& P = *pf;
  P = Prefilter();
  // ---- full factors + deduplicated byte sets
  std::map<ByteSet, uint16_t> set_ids;
  auto set_id = [&](const ByteSet& b) {
    auto it = set_ids.find(b); if (it != set_ids.end()) return it->second;
    uint16_t id = (uint16_t)set_ids.size(); set_ids.emplace(b, id);
    for (int k = 0; k < 8; k++) P.bytesets.push_back((uint32_t)(b.w[k >> 1] >> (32 * (k & 1))));
    return id;
  };
  std::vector<FactorSeq> seqs;          // parallel to P.factors
  for (size_t r = 0; r < rules.size(); r++) {
    if (rules[r].status != RULE_OK) continue;
    if (rules[r].factors.empty()) { P.always_rules.push_back((uint32_t)r); continue; }
    for (auto& f : rules[r].factors) {
      FullFactor ff{}; ff.rule = (uint32_t)r; ff.len = (uint8_t)std::min<size_t>(f.size(), kMaxFactorElems);
      ff.exact = (rules[r].factors_exact && f.size() <= (size_t)kMaxFactorElems) ? 1 : 0;
      ff.pre = rules[r].factor_pre >= 0xffff ? 0xffff : (uint16_t)rules[r].factor_pre;
      ff.pre_alpha = set_id(rules[r].factor_pre_alpha);
      for (int k = 0; k < ff.len; k++) ff.elem[k] = set_id(f[k]);
      P.factors.push_back(ff); seqs.push_back(FactorSeq(f.begin(), f.begin() + ff.len));
    }
  }
  if (P.factors.size() >= (1u << 20)) { if (err) *err = "too many factors"; return false; }
  const size_t nf = seqs.size();
  // folded images of every element
  std::vector<uint32_t> wild; { std::set<uint32_t> u; for (int b = 0; b < 256; b++) u.insert(gram_fold((uint32_t)b)); wild.assign(u.begin(), u.end()); }
  std::vector<std::vector<std::vector<uint32_t>>> img(nf);
  std::vector<std::vector<double>> eprob(nf);
  for (size_t f = 0; f < nf; f++) for (auto& e : seqs[f]) {
    std::set<uint32_t> u; double q = 0;
    for (int b = 0; b < 256; b++) if (e.has(b)) { u.insert(gram_fold((uint32_t)b)); q += Compiler::byte_weight(b); }
    img[f].push_back(std::vector<uint32_t>(u.begin(), u.end())); eprob[f].push_back(std::min(q, 1.0));
  }
  // best gram position of factor f for start residue r at stride S
  auto choose = [&](size_t f, int S, int r) {
    GramChoice best; const int L = (int)seqs[f].size();
    for (int o = -(kGramLen - 1); o <= L - 1; o++) {
      if ((((o + r) % S) + S) % S != 0) continue;
      double cnt = 1, p = 1; int inside = 0;
      for (int j = 0; j < kGramLen; j++) { int k = o + j; if (k < 0 || k >= L) cnt *= (double)wild.size(); else { cnt *= (double)img[f][k].size(); p *= eprob[f][k]; inside++; } }
      if (cnt < best.count || (cnt == best.count && (p < best.prob || (p == best.prob && inside > best.inside)))) { best.off = o; best.count = cnt; best.prob = p; best.inside = inside; }
    }
    best.ok = best.count <= (double)opt.max_keys_per_gram;
    return best;
  };
  auto plan = [&](int S, std::vector<std::vector<GramChoice>>* out, std::vector<char>* uncovered) {
    double total = 0; out->assign(nf, {}); uncovered->assign(nf, 0);
    for (size_t f = 0; f < nf; f++) {
      for (int r = 0; r < S; r++) { GramChoice c = choose(f, S, r); (*out)[f].push_back(c); if (!c.ok) (*uncovered)[f] = 1; }
      if (!(*uncovered)[f]) for (auto& c : (*out)[f]) total += c.count;
    }
    return total;
  };
  std::vector<std::vector<GramChoice>> ch; std::vector<char> unc;
  int S = opt.stride == 2 ? 2 : 4;
  double total = plan(S, &ch, &unc);
  if (S == 4 && opt.stride != 4) {
    // stride 4 needs every factor covered at four residues; one uncoverable short factor (or too many keys) moves the
    // whole set to stride 2, where the remaining uncoverable ones become triggers / always-candidates
    bool any_unc = false; for (char u : unc) any_unc |= u != 0;
    if (any_unc || total > (double)opt.max_keys) {
      std::vector<std::vector<GramChoice>> ch2; std::vector<char> unc2;
      double total2 = plan(2, &ch2, &unc2);
      size_t n4 = 0, n2 = 0; for (char u : unc) n4 += u != 0; for (char u : unc2) n2 += u != 0;
      if (n2 < n4 || total > (double)opt.max_keys) { S = 2; ch.swap(ch2); unc.swap(unc2); total = total2; }
    }
  }
  P.stride = S;
  // ---- factors no gram covers: single-byte trigger (rarest singleton element), else every message is a candidate
  std::vector<std::vector<uint32_t>> trig_lists;
  std::set<uint32_t> always(P.always_rules.begin(), P.always_rules.end());
  for (size_t f = 0; f < nf; f++) {
    if (!unc[f]) continue;
    int tk = -1, tb = -1; double tp = 2;
    for (int k = 0; k < (int)seqs[f].size(); k++) {
      int cnt = 0, last = -1; for (int b = 0; b < 256; b++) if (seqs[f][k].has(b)) { cnt++; last = b; }
      if (cnt == 1 && Compiler::byte_weight(last) < tp) { tp = Compiler::byte_weight(last); tk = k; tb = last; }
    }
    size_t ti = 0;
    if (tk >= 0) for (; ti < P.trig_bytes.size(); ti++) if (P.trig_bytes[ti] == (uint32_t)tb) break;
    if (tk < 0 || (ti == P.trig_bytes.size() && P.trig_bytes.size() >= 2)) { always.insert(P.factors[f].rule); continue; }
    if (ti == P.trig_bytes.size()) { P.trig_bytes.push_back((uint32_t)tb); trig_lists.emplace_back(); }
    trig_lists[ti].push_back((uint32_t)f | ((uint32_t)tk << 20));
  }
  P.always_rules.assign(always.begin(), always.end());
  // A rule that is a candidate for every message is verified over the whole message anyway: its factors leave the filter
  // altogether (an occurrence event would only shadow the whole-message run in the per-message candidate bitmap).
  std::vector<uint32_t> new_id(nf, 0xffffffffu);
  {
    std::vector<FullFactor> kept;
    for (size_t f = 0; f < nf; f++) if (!always.count(P.factors[f].rule)) { new_id[f] = (uint32_t)kept.size(); kept.push_back(P.factors[f]); }
    P.factors.swap(kept);
  }
  P.trig_offsets.assign(1, 0);
  for (auto& tl : trig_lists) {
    for (uint32_t e : tl) if (new_id[e & 0xfffffu] != 0xffffffffu) P.trig_list.push_back(new_id[e & 0xfffffu] | (e & 0xfff00000u));
    P.trig_offsets.push_back((uint32_t)P.trig_list.size());
  }
  // ---- keys + level-1b entries
  std::set<uint32_t> shapes;
  for (size_t f = 0; f < nf; f++) {
    if (unc[f] || new_id[f] == 0xffffffffu) continue;
    const int L = (int)seqs[f].size();
    for (int r = 0; r < S; r++) {
      const GramChoice& c = ch[f][r];
      GramEntry e{}; e.factor = new_id[f]; e.off = c.off;
      std::vector<uint32_t> cur = {0};
      for (int j = 0; j < kGramLen; j++) {
        const int k = c.off + j; const std::vector<uint32_t>& opts = (k < 0 || k >= L) ? wild : img[f][k];
        if (k >= 0 && k < L && opts.size() == 1) { e.key |= opts[0] << (8 * j); e.mask |= 0xffu << (8 * j); }
        std::vector<uint32_t> nx; nx.reserve(cur.size() * opts.size());
        for (uint32_t base : cur) for (uint32_t v : opts) nx.push_back(base | (v << (8 * j)));
        cur.swap(nx);
      }
      P.keys.insert(P.keys.end(), cur.begin(), cur.end());
      P.entries.push_back(e); shapes.insert(e.mask);
    }
  }
  std::sort(P.keys.begin(), P.keys.end()); P.keys.erase(std::unique(P.keys.begin(), P.keys.end()), P.keys.end());
  P.shapes.assign(shapes.begin(), shapes.end());
  P.min_factor_len = 255; P.max_factor_len = 0;
  for (auto& ff : P.factors) { P.min_factor_len = std::min<uint32_t>(P.min_factor_len, ff.len); P.max_factor_len = std::max<uint32_t>(P.max_factor_len, ff.len); }
  if (P.factors.empty()) P.min_factor_len = 0;
  (void)err;
  return true;
}

// ---------------------------------------------------------------------------------------------------------------
// bit-parallel form of a Pike program (bitprog.h)
bool build_bitprog(const CompiledRule& r, std::vector<uint64_t>* outv) {
  const std::vector<uint32_t>& prog = r.prog;
  if (r.status != RULE_OK || prog.empty()) return false;
  std::vector<int> bit_of(prog.size(), -1); int nc = 0;
  int lb_set = -1, la_set = -1;                     // the rule's lookbehind / lookahead set (one per direction, ASCII-only)
  for (size_t pc = 0; pc < prog.size(); pc++) {
    const uint32_t op = prog[pc] & 0xff, arg = prog[pc] >> 8;
    if (op == OP_CHAR || op == OP_SET || op == OP_ANY) { if (nc >= 127) return false; bit_of[pc] = nc++; }
    else if (op == OP_LOOKAHEAD || op == OP_NLOOKAHEAD || op == OP_LOOKBEHIND || op == OP_NLOOKBEHIND) {
      if (arg >= r.sets.size() || !r.sets[arg].ranges.empty()) return false;      // a set with non-ASCII members: the byte walk cannot evaluate it
      int& slot = (op == OP_LOOKBEHIND || op == OP_NLOOKBEHIND) ? lb_set : la_set;
      if (slot >= 0 && !(r.sets[slot] == r.sets[arg])) return false;
      if (slot < 0) slot = (int)arg;
    }
  }
  const uint32_t W = nc <= 63 ? 1u : 2u, match_bit = 64 * W - 1;
  struct Mask { uint64_t w[2] = {0, 0}; void set(uint32_t b) { w[b >> 6] |= 1ull << (b & 63); } bool has(uint32_t b) const { return (w[b >> 6] >> (b & 63)) & 1; }
                bool operator==(const Mask& o) const { return w[0] == o.w[0] && w[1] == o.w[1]; } bool zero() const { return !(w[0] | w[1]); } };
  const bool has_look = lb_set >= 0 || la_set >= 0;
  // closure of the epsilon edges from pc under context ctx: bit 0 word boundary, bit 1 start of message, bit 2 end, bit 3 previous
  // unit in the lookbehind set, bit 4 next unit in the lookahead set
  auto closure = [&](uint32_t pc0, uint32_t ctx) {
    Mask m; std::vector<char> seen(prog.size(), 0); std::vector<uint32_t> st{pc0};
    while (!st.empty()) {
      uint32_t pc = st.back(); st.pop_back();
      if (pc >= prog.size() || seen[pc]) continue;
      seen[pc] = 1;
      const uint32_t op = prog[pc] & 0xff, arg = prog[pc] >> 8;
      switch (op) {
        case OP_SPLIT_NEXT: case OP_SPLIT_JUMP: st.push_back(pc + 1); st.push_back(arg); break;
        case OP_JMP: case OP_JMP_BACK: st.push_back(arg); break;
        case OP_EMPTYCHK: st.push_back(pc + 1); break;
        case OP_BOL: if (ctx & 2u) st.push_back(pc + 1); break;
        case OP_EOL: if (ctx & 4u) st.push_back(pc + 1); break;
        case OP_WORDB: if (ctx & 1u) st.push_back(pc + 1); break;
        case OP_NWORDB: if (!(ctx & 1u)) st.push_back(pc + 1); break;
        case OP_LOOKBEHIND: if (ctx & 8u) st.push_back(pc + 1); break;
        case OP_NLOOKBEHIND: if (!(ctx & 8u)) st.push_back(pc + 1); break;
        case OP_LOOKAHEAD: if (ctx & 16u) st.push_back(pc + 1); break;
        case OP_NLOOKAHEAD: if (!(ctx & 16u)) st.push_back(pc + 1); break;
        case OP_MATCH: m.set(match_bit); break;
        default: m.set((uint32_t)bit_of[pc]); break;
      }
    }
    return m;
  };
  // layout: bitprog.h
  std::vector<uint64_t>& out = *outv;
  const uint32_t n_ctx = 32, meta_off = 1 + (128 + n_ctx) * W, rows_off = meta_off + 7 + 2 * W;
  out.assign(rows_off, 0);
  out[0] = W;
  for (size_t pc = 0; pc < prog.size(); pc++) {
    if (bit_of[pc] < 0) continue;
    const uint32_t op = prog[pc] & 0xff, arg = prog[pc] >> 8, k = (uint32_t)bit_of[pc];
    for (int b = 0; b < 128; b++) {
      bool ok = op == OP_CHAR ? (uint32_t)b == arg : op == OP_ANY ? !(b == 0x0a || b == 0x0d) : ((r.sets[arg].ascii[b >> 5] >> (b & 31)) & 1u) != 0;
      if (ok) out[1 + (size_t)b * W + (k >> 6)] |= 1ull << (k & 63);
    }
  }
  std::vector<std::vector<Mask>> rows; uint64_t rowmap[2] = {0, 0};
  bool start_same = true; Mask start_first;
  for (uint32_t ctx = 0; ctx < n_ctx; ctx++) {
    std::vector<Mask> row(64 * W);
    for (size_t pc = 0; pc < prog.size(); pc++) if (bit_of[pc] >= 0) row[bit_of[pc]] = closure((uint32_t)pc + 1, ctx);
    const Mask st = closure(0, ctx);
    for (uint32_t w = 0; w < W; w++) out[1 + (128 + ctx) * W + w] = st.w[w];
    if (ctx == 0) start_first = st; else start_same = start_same && st == start_first;
    uint32_t ri = 0;
    while (ri < rows.size() && !(rows[ri] == row)) ri++;
    if (ri == rows.size()) { if (rows.size() >= 15) return false; rows.push_back(row); }
    rowmap[ctx >> 4] |= (uint64_t)ri << (4 * (ctx & 15));
  }
  const uint32_t n_rows = (uint32_t)rows.size();
  out[meta_off] = n_rows | ((uint64_t)W << 4) | (start_same ? 1ull << 8 : 0) | (has_look ? 1ull << 9 : 0);
  out[meta_off + 1] = rowmap[0]; out[meta_off + 2] = rowmap[1];
  auto set128 = [&](int sid, uint64_t* o) { o[0] = o[1] = 0; if (sid >= 0) { o[0] = (uint64_t)r.sets[sid].ascii[0] | ((uint64_t)r.sets[sid].ascii[1] << 32); o[1] = (uint64_t)r.sets[sid].ascii[2] | ((uint64_t)r.sets[sid].ascii[3] << 32); } };
  set128(lb_set, &out[meta_off + 3]); set128(la_set, &out[meta_off + 5]);
  // instructions whose successors are {k + 1} and / or {k} in every row: a shift and a mask instead of a table row
  for (int k = 0; k < nc; k++) {
    const Mask f = rows[0][k];
    Mask rest = f; rest.w[k >> 6] &= ~(1ull << (k & 63)); rest.w[(k + 1) >> 6] &= ~(1ull << ((k + 1) & 63));
    bool simple = rest.zero();
    for (uint32_t ri = 1; ri < n_rows && simple; ri++) simple = rows[ri][k] == f;
    if (!simple) continue;
    if (f.has(k + 1)) out[meta_off + 7 + (k >> 6)] |= 1ull << (k & 63);
    if (f.has(k)) out[meta_off + 7 + W + (k >> 6)] |= 1ull << (k & 63);
  }
  for (uint32_t ri = 0; ri < n_rows; ri++) for (uint32_t k = 0; k < 64 * W; k++) for (uint32_t w = 0; w < W; w++) out.push_back(rows[ri][k].w[w]);
  return true;
}

}  // namespace cg
