// regex.cpp -- a regular expression over UTF-8 text -> a trimmed, minimal byte-level DFA (DESIGN.md §9g).
//
// parse (code point sets, concatenation, alternation, counted repetition) -> Thompson NFA over bytes (each code point set
// as the byte-range sequences of its UTF-8 encodings) -> subset construction over byte classes -> trimming (states that
// cannot reach an accepting state become -1) -> minimisation (Valmari and Lehtinen's partition refinement, O(m log n)) ->
// states renumbered breadth-first from the start, which is state 0.
#include "regex.hpp"

#include <algorithm>
#include <cstdio>
#include <map>
#include <utility>

namespace lnb {
namespace {

constexpr int kMaxNfa = 1 << 20;       // NFA nodes a pattern may expand to (counted repetition copies its operand)
constexpr int kMaxSubset = 1 << 17;    // DFA states of the subset construction, before trimming and minimisation
constexpr int kMaxCount = 100000;      // the largest m, n of {m}, {m,}, {m,n}
constexpr int kMaxDepth = 1000;        // nested groups (the parser and the NFA builder recurse once per level)
constexpr uint32_t kMaxCp = 0x10FFFF;

struct Error {
  std::string msg;
};
[[noreturn]] void bad(int64_t off, const char* what) {
  char b[256];
  snprintf(b, sizeof b, "regex: %s at byte offset %lld", what, (long long)off);
  throw Error{b};
}

using Ranges = std::vector<std::pair<uint32_t, uint32_t>>;   // closed code point ranges

Ranges normalize(Ranges r) {
  std::sort(r.begin(), r.end());
  Ranges o;
  for (auto& x : r) {
    if (!o.empty() && x.first <= o.back().second + 1) o.back().second = std::max(o.back().second, x.second);
    else o.push_back(x);
  }
  return o;
}
Ranges complement(const Ranges& in) {
  Ranges r = normalize(in), o;
  uint32_t lo = 0;
  for (auto& x : r) {
    if (x.first > lo) o.push_back({lo, x.first - 1});
    lo = x.second + 1;
  }
  if (lo <= kMaxCp) o.push_back({lo, kMaxCp});
  return o;
}
// UTF-8 cannot encode the surrogates U+D800..U+DFFF: no string of the language contains them
Ranges encodable(const Ranges& in) {
  Ranges o;
  for (auto& x : normalize(in)) {
    if (x.second < 0xD800 || x.first > 0xDFFF) { o.push_back(x); continue; }
    if (x.first < 0xD800) o.push_back({x.first, 0xD7FF});
    if (x.second > 0xDFFF) o.push_back({0xE000, x.second});
  }
  return o;
}

// ---- syntax tree -------------------------------------------------------------------------------------------------------
struct Node {
  enum Kind { EMPTY, SET, CAT, ALT, REP } kind;
  Ranges set;
  std::vector<int> kids;
  int mn = 0, mx = 0;   // REP: mx -1 = unbounded
};

struct Parser {
  const unsigned char* p;
  int64_t n, i = 0;
  std::vector<Node> nodes;
  int depth = 0;

  int add(Node x) { nodes.push_back(std::move(x)); return (int)nodes.size() - 1; }
  int set_node(Ranges r) { Node x{Node::SET, encodable(r), {}, 0, 0}; return add(std::move(x)); }

  // one UTF-8 encoded code point at i
  uint32_t code_point() {
    const int64_t at = i;
    const unsigned c = p[i];
    int len = c < 0x80 ? 1 : (c >> 5) == 6 ? 2 : (c >> 4) == 14 ? 3 : (c >> 3) == 30 ? 4 : 0;
    if (!len || i + len > n) bad(at, "invalid UTF-8");
    uint32_t v = len == 1 ? c : len == 2 ? (c & 0x1F) : len == 3 ? (c & 0x0F) : (c & 0x07);
    for (int k = 1; k < len; k++) {
      if ((p[i + k] & 0xC0) != 0x80) bad(at, "invalid UTF-8");
      v = (v << 6) | (p[i + k] & 0x3F);
    }
    static const uint32_t min_of_len[5] = {0, 0, 0x80, 0x800, 0x10000};
    if (v < min_of_len[len] || v > kMaxCp || (v >= 0xD800 && v <= 0xDFFF)) bad(at, "invalid UTF-8");
    i += len;
    return v;
  }
  uint32_t hex(int digits, int64_t at) {
    uint32_t v = 0;
    for (int k = 0; k < digits; k++, i++) {
      if (i >= n) bad(at, "incomplete escape");
      const int c = p[i];
      const int d = c >= '0' && c <= '9' ? c - '0' : c >= 'a' && c <= 'f' ? c - 'a' + 10 : c >= 'A' && c <= 'F' ? c - 'A' + 10 : -1;
      if (d < 0) bad(at, "incomplete escape");
      v = v * 16 + d;
    }
    return v;
  }
  // an escape at i (p[i] == '\\'): a single code point (returns true, *cp) or a shorthand set (*set)
  bool escape(uint32_t* cp, Ranges* set) {
    const int64_t at = i++;
    if (i >= n) bad(at, "trailing backslash");
    const int c = p[i++];
    const Ranges digit = {{'0', '9'}}, word = {{'0', '9'}, {'A', 'Z'}, {'_', '_'}, {'a', 'z'}}, space = {{'\t', '\r'}, {' ', ' '}};
    switch (c) {
      case 'd': *set = digit; return false;
      case 'D': *set = complement(digit); return false;
      case 'w': *set = word; return false;
      case 'W': *set = complement(word); return false;
      case 's': *set = space; return false;
      case 'S': *set = complement(space); return false;
      case 'n': *cp = '\n'; return true;
      case 't': *cp = '\t'; return true;
      case 'r': *cp = '\r'; return true;
      case 'f': *cp = '\f'; return true;
      case 'v': *cp = '\v'; return true;
      case 'x': *cp = hex(2, at); return true;
      case 'u': *cp = hex(4, at); return true;
      default: break;
    }
    if (c >= '0' && c <= '9') bad(at, "backreferences and octal escapes are not supported");
    if (c == 'b' || c == 'B' || c == 'A' || c == 'Z') bad(at, "anchors are not supported");
    if ((c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || c >= 0x80) bad(at, "unsupported escape");
    *cp = (uint32_t)c;   // an escaped ASCII punctuation or space character stands for itself
    return true;
  }

  int alt() {
    std::vector<int> kids{cat()};
    while (i < n && p[i] == '|') { i++; kids.push_back(cat()); }
    if (kids.size() == 1) return kids[0];
    Node x{Node::ALT, {}, std::move(kids), 0, 0};
    return add(std::move(x));
  }
  int cat() {
    std::vector<int> kids;
    while (i < n && p[i] != '|' && p[i] != ')') kids.push_back(repeat());
    if (kids.empty()) return add(Node{Node::EMPTY, {}, {}, 0, 0});
    if (kids.size() == 1) return kids[0];
    Node x{Node::CAT, {}, std::move(kids), 0, 0};
    return add(std::move(x));
  }
  int number(int64_t at) {
    if (i >= n || p[i] < '0' || p[i] > '9') bad(at, "unsupported '{' (a repeat is {m}, {m,} or {m,n})");
    long long v = 0;
    while (i < n && p[i] >= '0' && p[i] <= '9') {
      v = v * 10 + (p[i++] - '0');
      if (v > kMaxCount) bad(at, "repeat count above 100000");
    }
    return (int)v;
  }
  int repeat() {
    int a = atom();
    if (i >= n || !(p[i] == '*' || p[i] == '+' || p[i] == '?' || p[i] == '{')) return a;
    const int64_t at = i;
    int mn, mx;
    const int c = p[i++];
    if (c == '*') { mn = 0; mx = -1; }
    else if (c == '+') { mn = 1; mx = -1; }
    else if (c == '?') { mn = 0; mx = 1; }
    else {
      mn = mx = number(at);
      if (i < n && p[i] == ',') {
        i++;
        mx = (i < n && p[i] == '}') ? -1 : number(at);
      }
      if (i >= n || p[i] != '}') bad(at, "unsupported '{' (a repeat is {m}, {m,} or {m,n})");
      i++;
      if (mx >= 0 && mn > mx) bad(at, "min repeat greater than max repeat");
    }
    if (i < n && p[i] == '?') i++;   // lazy: the same language
    if (i < n && (p[i] == '*' || p[i] == '+' || p[i] == '?' || p[i] == '{'))
      bad(i, p[i] == '+' ? "possessive repeats are not supported" : "multiple repeat");
    Node x{Node::REP, {}, {a}, mn, mx};
    return add(std::move(x));
  }
  int atom() {
    const int64_t at = i;
    const int c = p[i];
    if (c == '(') {
      if (++depth > kMaxDepth) bad(at, "groups nested deeper than 1000");
      i++;
      if (i < n && p[i] == '?') {
        if (i + 1 < n && p[i + 1] == ':') i += 2;
        else bad(at, "unsupported group (only (...) and (?:...) are supported)");
      }
      const int r = alt();
      if (i >= n || p[i] != ')') bad(at, "missing ), unterminated subpattern");
      i++;
      depth--;
      return r;
    }
    if (c == '[') return cls();
    if (c == '.') { i++; return set_node(complement({{'\n', '\n'}})); }
    if (c == '^' || c == '$') bad(at, "anchors are not supported");
    if (c == '*' || c == '+' || c == '?' || c == '{') bad(at, "nothing to repeat");
    if (c == '\\') {
      uint32_t cp = 0;
      Ranges s;
      return escape(&cp, &s) ? set_node({{cp, cp}}) : set_node(s);
    }
    const uint32_t cp = code_point();
    return set_node({{cp, cp}});
  }
  // one member of a class at i: a code point (true, *cp) or a shorthand set
  bool class_atom(uint32_t* cp, Ranges* set) {
    if (p[i] == '\\') return escape(cp, set);
    *cp = code_point();
    return true;
  }
  int cls() {
    const int64_t at = i++;
    bool neg = false;
    if (i < n && p[i] == '^') { neg = true; i++; }
    Ranges r;
    bool first = true;
    for (;;) {
      if (i >= n) bad(at, "unterminated character set");
      if (p[i] == ']' && !first) { i++; break; }
      first = false;
      const int64_t item = i;
      uint32_t lo = 0, hi = 0;
      Ranges s;
      if (!class_atom(&lo, &s)) {
        if (i + 1 < n && p[i] == '-' && p[i + 1] != ']') bad(item, "bad character range");
        r.insert(r.end(), s.begin(), s.end());
        continue;
      }
      if (i + 1 < n && p[i] == '-' && p[i + 1] != ']') {
        i++;
        if (!class_atom(&hi, &s)) bad(item, "bad character range");
        if (hi < lo) bad(item, "bad character range");
      } else {
        hi = lo;
      }
      r.push_back({lo, hi});
    }
    return set_node(neg ? complement(r) : r);
  }
};

// ---- Thompson NFA over bytes -------------------------------------------------------------------------------------------
struct Nfa {
  struct Edge { uint8_t lo, hi; int to; };
  std::vector<std::vector<Edge>> edges;
  std::vector<std::vector<int>> eps;
  int add() {
    if ((int)edges.size() >= kMaxNfa) throw Error{"regex: the pattern expands to more than 1048576 NFA states"};
    edges.emplace_back();
    eps.emplace_back();
    return (int)edges.size() - 1;
  }
};

// the byte-range sequences of the UTF-8 encodings of [lo, hi] (no surrogates inside), each a product of byte ranges
void utf8_sequences(uint32_t lo, uint32_t hi, std::vector<std::vector<std::pair<uint8_t, uint8_t>>>& out) {
  static const uint32_t bounds[3] = {0x7F, 0x7FF, 0xFFFF};
  for (uint32_t b : bounds)
    if (lo <= b && hi > b) { utf8_sequences(lo, b, out); utf8_sequences(b + 1, hi, out); return; }
  if (hi < 0x80) { out.push_back({{(uint8_t)lo, (uint8_t)hi}}); return; }
  for (int k = 1; k < 4; k++) {
    const uint32_t m = (1u << (6 * k)) - 1;
    if ((lo & ~m) != (hi & ~m)) {
      if ((lo & m) != 0) { utf8_sequences(lo, lo | m, out); utf8_sequences((lo | m) + 1, hi, out); return; }
      if ((hi & m) != m) { utf8_sequences(lo, (hi & ~m) - 1, out); utf8_sequences(hi & ~m, hi, out); return; }
    }
  }
  auto enc = [](uint32_t v, uint8_t* b) -> int {
    if (v < 0x800) { b[0] = 0xC0 | (v >> 6); b[1] = 0x80 | (v & 0x3F); return 2; }
    if (v < 0x10000) { b[0] = 0xE0 | (v >> 12); b[1] = 0x80 | ((v >> 6) & 0x3F); b[2] = 0x80 | (v & 0x3F); return 3; }
    b[0] = 0xF0 | (v >> 18); b[1] = 0x80 | ((v >> 12) & 0x3F); b[2] = 0x80 | ((v >> 6) & 0x3F); b[3] = 0x80 | (v & 0x3F);
    return 4;
  };
  uint8_t a[4], b[4];
  const int len = enc(lo, a);
  enc(hi, b);
  std::vector<std::pair<uint8_t, uint8_t>> seq;
  for (int k = 0; k < len; k++) seq.push_back({a[k], b[k]});
  out.push_back(seq);
}

struct Frag { int in, out; };

Frag emit(const std::vector<Node>& t, int id, Nfa& a) {
  const Node& x = t[id];
  switch (x.kind) {
    case Node::EMPTY: { const int s = a.add(); return {s, s}; }
    case Node::SET: {
      const int s = a.add(), e = a.add();
      std::vector<std::vector<std::pair<uint8_t, uint8_t>>> seqs;
      for (auto& r : x.set) utf8_sequences(r.first, r.second, seqs);
      for (auto& q : seqs) {
        int cur = s;
        for (size_t k = 0; k < q.size(); k++) {
          const int nx = k + 1 == q.size() ? e : a.add();
          a.edges[cur].push_back({q[k].first, q[k].second, nx});
          cur = nx;
        }
      }
      return {s, e};
    }
    case Node::CAT: {
      Frag f = emit(t, x.kids[0], a);
      for (size_t k = 1; k < x.kids.size(); k++) {
        const Frag g = emit(t, x.kids[k], a);
        a.eps[f.out].push_back(g.in);
        f.out = g.out;
      }
      return f;
    }
    case Node::ALT: {
      const int s = a.add(), e = a.add();
      for (int k : x.kids) {
        const Frag g = emit(t, k, a);
        a.eps[s].push_back(g.in);
        a.eps[g.out].push_back(e);
      }
      return {s, e};
    }
    case Node::REP: {
      const int s = a.add();
      int cur = s;
      for (int k = 0; k < x.mn; k++) {
        const Frag g = emit(t, x.kids[0], a);
        a.eps[cur].push_back(g.in);
        cur = g.out;
      }
      if (x.mx < 0) {   // cur loops through one more copy
        const Frag g = emit(t, x.kids[0], a);
        a.eps[cur].push_back(g.in);
        a.eps[g.out].push_back(cur);
        return {s, cur};
      }
      const int e = a.add();
      for (int k = x.mn; k < x.mx; k++) {
        const Frag g = emit(t, x.kids[0], a);
        a.eps[cur].push_back(e);
        a.eps[cur].push_back(g.in);
        cur = g.out;
      }
      a.eps[cur].push_back(e);
      return {s, e};
    }
  }
  return {0, 0};
}

// ---- minimisation: Valmari and Lehtinen's refinable partitions ---------------------------------------------------------
struct Partition {
  int z = 0;
  std::vector<int> E, L, S, F, P;   // elements by set, location of each element, set of each, set [F, P) in E
  void init(int n) {
    z = n > 0 ? 1 : 0;
    E.resize(n); L.resize(n); S.assign(n, 0); F.assign(n + 1, 0); P.assign(n + 1, 0);
    for (int i = 0; i < n; i++) E[i] = L[i] = i;
    if (z) P[0] = n;
  }
  std::vector<int> M, W;
  void mark(int e) {
    const int s = S[e], i = L[e], j = F[s] + M[s];
    E[i] = E[j]; L[E[i]] = i; E[j] = e; L[e] = j;
    if (!M[s]++) W.push_back(s);
  }
  void split() {
    while (!W.empty()) {
      const int s = W.back();
      W.pop_back();
      const int j = F[s] + M[s];
      if (j == P[s]) { M[s] = 0; continue; }
      if (M[s] <= P[s] - j) { F[z] = F[s]; P[z] = F[s] = j; }
      else { P[z] = P[s]; F[z] = P[s] = j; }
      for (int i = F[z]; i < P[z]; i++) S[E[i]] = z;
      M[s] = M[z++] = 0;
    }
  }
};

}  // namespace

bool regex_dfa(const char* pattern, int64_t len, int max_states, std::vector<int32_t>& trans, std::vector<uint8_t>& accept,
               std::string& err, int* n_states) {
  if (n_states) *n_states = 0;
  try {
    Parser ps{reinterpret_cast<const unsigned char*>(pattern), len, 0, {}, 0};
    const int root = ps.alt();
    if (ps.i < len) bad(ps.i, "unbalanced parenthesis");
    Nfa nfa;
    const Frag top = emit(ps.nodes, root, nfa);
    const int nn = (int)nfa.edges.size(), fin = top.out;

    // byte classes: bytes no NFA edge tells apart share a class
    std::vector<uint8_t> cut(257, 0);
    for (auto& es : nfa.edges)
      for (auto& e : es) { cut[e.lo] = 1; cut[e.hi + 1] = 1; }
    int cls[256], k = -1;
    std::vector<int> rep;
    for (int b = 0; b < 256; b++) {
      if (b == 0 || cut[b]) { k++; rep.push_back(b); }
      cls[b] = k;
    }
    const int K = k + 1;

    // subset construction
    std::vector<int> stamp(nn, -1), stack;
    int clock = 0;
    auto closure = [&](std::vector<int>& v) {
      clock++;
      stack.assign(v.begin(), v.end());
      v.clear();
      for (int x : stack) stamp[x] = clock;
      while (!stack.empty()) {
        const int x = stack.back();
        stack.pop_back();
        v.push_back(x);
        for (int y : nfa.eps[x])
          if (stamp[y] != clock) { stamp[y] = clock; stack.push_back(y); }
      }
      std::sort(v.begin(), v.end());
    };
    std::map<std::vector<int>, int> ids;
    std::vector<std::vector<int>> sets;
    std::vector<int> dt;   // [state][K]
    std::vector<uint8_t> acc;
    std::vector<int> start{top.in};
    closure(start);
    ids[start] = 0;
    sets.push_back(start);
    for (size_t q = 0; q < sets.size(); q++) {
      acc.push_back(std::binary_search(sets[q].begin(), sets[q].end(), fin) ? 1 : 0);
      for (int c = 0; c < K; c++) {
        const int b = rep[c];
        std::vector<int> nx;
        clock++;
        for (int x : sets[q])
          for (auto& e : nfa.edges[x])
            if (b >= e.lo && b <= e.hi && stamp[e.to] != clock) { stamp[e.to] = clock; nx.push_back(e.to); }
        if (nx.empty()) { dt.push_back(-1); continue; }
        closure(nx);
        auto it = ids.find(nx);
        if (it != ids.end()) { dt.push_back(it->second); continue; }
        if ((int)sets.size() >= kMaxSubset) throw Error{"regex: the subset construction passes 131072 DFA states"};
        const int id = (int)sets.size();
        ids.emplace(nx, id);
        sets.push_back(std::move(nx));
        dt.push_back(id);
      }
    }
    const int nd = (int)sets.size();
    sets.clear();
    ids.clear();

    // trimming: keep the states that reach an accepting state
    std::vector<std::vector<int>> pred(nd);
    for (int q = 0; q < nd; q++)
      for (int c = 0; c < K; c++)
        if (dt[q * K + c] >= 0) pred[dt[q * K + c]].push_back(q);
    std::vector<uint8_t> live(nd, 0);
    for (int q = 0; q < nd; q++)
      if (acc[q]) { live[q] = 1; stack.push_back(q); }
    while (!stack.empty()) {
      const int q = stack.back();
      stack.pop_back();
      for (int r : pred[q])
        if (!live[r]) { live[r] = 1; stack.push_back(r); }
    }
    if (!live[0]) throw Error{"regex: the pattern matches no string"};

    // minimisation over the live states; transitions into dead states are absent (partial DFA)
    std::vector<int> tail, label, head;
    for (int q = 0; q < nd; q++)
      if (live[q])
        for (int c = 0; c < K; c++) {
          const int r = dt[q * K + c];
          if (r >= 0 && live[r]) { tail.push_back(q); label.push_back(c); head.push_back(r); }
        }
    const int m = (int)tail.size();
    Partition B, C;
    B.init(nd);
    B.M.assign(nd + 1, 0);
    for (int q = 0; q < nd; q++)
      if (!live[q]) B.mark(q);
    B.split();   // dead states form their own set, never a splitter's tail
    for (int q = 0; q < nd; q++)
      if (live[q] && acc[q]) B.mark(q);
    B.split();
    C.init(m);
    C.M.assign(m + 1, 0);
    if (m) {   // transitions split by label
      std::vector<int> order(m);
      for (int i = 0; i < m; i++) order[i] = i;
      std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return label[x] < label[y]; });
      for (int i = 0; i < m; i++) { C.E[i] = order[i]; C.L[order[i]] = i; }
      C.z = 0;
      for (int i = 0; i < m; i++) {
        if (i == 0 || label[order[i]] != label[order[i - 1]]) { C.F[C.z] = i; C.z++; }
        C.S[order[i]] = C.z - 1;
        C.P[C.z - 1] = i + 1;
      }
    }
    std::vector<int> in_off(nd + 1, 0), in_tr(m);   // incoming transitions of each state
    for (int t = 0; t < m; t++) in_off[head[t] + 1]++;
    for (int q = 0; q < nd; q++) in_off[q + 1] += in_off[q];
    {
      std::vector<int> fill(in_off.begin(), in_off.end() - 1);
      for (int t = 0; t < m; t++) in_tr[fill[head[t]]++] = t;
    }
    for (int b = 1, c = 0; c < C.z;) {
      for (int i = C.F[c]; i < C.P[c]; i++) B.mark(tail[C.E[i]]);
      B.split();
      c++;
      for (; b < B.z; b++) {   // each new set splits the cords by whether a transition enters it
        for (int i = B.F[b]; i < B.P[b]; i++) {
          const int q = B.E[i];
          for (int j = in_off[q]; j < in_off[q + 1]; j++) C.mark(in_tr[j]);
        }
        C.split();
      }
    }

    // breadth-first numbering of the live sets from the start's
    std::vector<int> num(B.z, -1), order;
    std::vector<int> any(B.z, -1);   // a member state of each set
    for (int q = 0; q < nd; q++)
      if (live[q] && any[B.S[q]] < 0) any[B.S[q]] = q;
    num[B.S[0]] = 0;
    order.push_back(B.S[0]);
    for (size_t h = 0; h < order.size(); h++) {
      const int q = any[order[h]];
      for (int c = 0; c < K; c++) {
        const int r = dt[q * K + c];
        if (r < 0 || !live[r]) continue;
        const int s = B.S[r];
        if (num[s] < 0) { num[s] = (int)order.size(); order.push_back(s); }
      }
    }
    const int Q = (int)order.size();
    if (n_states) *n_states = Q;
    if (Q > max_states) {
      char b[160];
      snprintf(b, sizeof b, "regex: the minimal DFA has %d states, more than %d", Q, max_states);
      throw Error{b};
    }
    trans.assign((size_t)Q * 256, -1);
    accept.assign(Q, 0);
    for (int s = 0; s < Q; s++) {
      const int q = any[order[s]];
      accept[s] = acc[q];
      for (int b = 0; b < 256; b++) {
        const int r = dt[q * K + cls[b]];
        if (r >= 0 && live[r]) trans[(size_t)s * 256 + b] = num[B.S[r]];
      }
    }
    return true;
  } catch (const Error& e) {
    err = e.msg;
    return false;
  } catch (const std::bad_alloc&) {
    err = "regex: out of host memory";
    return false;
  }
}

}  // namespace lnb
