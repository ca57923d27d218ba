// The DBoW2 text vocabulary: a hand-written parser (ORBvoc.txt is 145 MB, about 39 M tokens), the tree checks, and the device copy.
// The format and every rule are stated in include/sivo_b200.h; oracle/bow_oracle.py restates the parser.
#include <cerrno>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <string>

#include "vocabulary.h"

namespace sivo {
namespace {

// the characters std::istream's >> skips (isspace in the C locale) other than the line break
inline bool is_blank(char c) { return c == ' ' || c == '\t' || c == '\r' || c == '\v' || c == '\f'; }

struct Tokens {
  const char* p;
  const char* end;
  // the next whitespace-separated token in [p, end), or false at the end of the line
  bool next(const char*& b, const char*& e) {
    while (p < end && is_blank(*p)) ++p;
    if (p == end) return false;
    b = p;
    while (p < end && !is_blank(*p)) ++p;
    e = p;
    return true;
  }
};

// a whole token that is a decimal integer within int
bool parse_int(const char* b, const char* e, int& out) {
  bool neg = false;
  if (b < e && (*b == '+' || *b == '-')) neg = *b++ == '-';
  if (b == e) return false;
  long long v = 0;
  for (; b < e; ++b) {
    if (*b < '0' || *b > '9') return false;
    v = v * 10 + (*b - '0');
    if (v > 2147483648ll) return false;
  }
  if (neg) v = -v;
  if (v > 2147483647ll || v < -2147483648ll) return false;
  out = static_cast<int>(v);
  return true;
}

// a whole token that strtod reads (std::istream's >> for a double reads the same text the same way)
bool parse_double(const char* b, const char* e, double& out) {
  char buf[128];
  const size_t len = static_cast<size_t>(e - b);
  if (len == 0 || len >= sizeof buf) return false;
  memcpy(buf, b, len);
  buf[len] = 0;
  char* stop = nullptr;
  errno = 0;
  out = strtod(buf, &stop);
  return stop == buf + len;
}

std::string read_file(const char* path) {
  FILE* f = fopen(path, "rb");
  if (!f) fail(SIVO_ENOENT, "vocabulary: cannot open %s", path);
  std::string s;
  char buf[1 << 16];
  size_t got;
  while ((got = fread(buf, 1, sizeof buf, f)) > 0) s.append(buf, got);
  const bool bad = ferror(f);
  fclose(f);
  if (bad) fail(SIVO_ENOENT, "vocabulary: cannot read %s", path);
  return s;
}

}  // namespace

void check_vocabulary(int k, int L, int scoring, int weighting, const int32_t* parent, const uint8_t* is_leaf, int n) {
  if (k < 0 || k > 20 || L < 1 || L > 10 || scoring < 0 || scoring > 5 || weighting < 0 || weighting > 3)
    fail(SIVO_EFORMAT, "vocabulary: header k %d L %d scoring %d weighting %d out of range", k, L, scoring, weighting);
  if (n < 2) fail(SIVO_EFORMAT, "vocabulary: empty tree");
  std::vector<int> n_children(n, 0);
  for (int i = 1; i < n; ++i) {
    const int p = parent[i];
    if (p < 0 || p >= i) fail(SIVO_EFORMAT, "vocabulary: node %d has parent %d, not an earlier node", i, p);
    if (p > 0 && is_leaf[p]) fail(SIVO_EFORMAT, "vocabulary: node %d has the leaf %d as its parent", i, p);
    ++n_children[p];
  }
  for (int i = 0; i < n; ++i)
    if ((i == 0 || !is_leaf[i]) && n_children[i] == 0) fail(SIVO_EFORMAT, "vocabulary: node %d is not a leaf and has no children", i);
}

void parse_vocabulary_text(const char* path, VocTree& t) {
  const std::string text = read_file(path);
  const char* p = text.data();
  const char* const end = p + text.size();
  // the next line [b, e) without its '\n'; false after the last one (a final '\n' ends the last line, it does not start one)
  auto next_line = [&](const char*& b, const char*& e) {
    if (p >= end) return false;
    b = p;
    const void* nl = memchr(p, '\n', static_cast<size_t>(end - p));
    e = nl ? static_cast<const char*>(nl) : end;
    p = nl ? e + 1 : end;
    return true;
  };
  const char *lb, *le, *tb, *te;
  if (!next_line(lb, le)) fail(SIVO_EFORMAT, "vocabulary: empty file");
  Tokens hdr{lb, le};
  int h[4];
  for (int i = 0; i < 4; ++i)
    if (!hdr.next(tb, te) || !parse_int(tb, te, h[i])) fail(SIVO_EFORMAT, "vocabulary: the header needs k L scoring weighting");
  t = VocTree{};
  t.k = h[0]; t.L = h[1]; t.scoring = h[2]; t.weighting = h[3];
  t.parent.assign(1, -1);
  t.is_leaf.assign(1, 0);
  t.desc.assign(32, 0);
  t.weight.assign(1, 0.0);
  int line = 1, blank_line = 0;
  while (next_line(lb, le)) {
    ++line;
    Tokens tok{lb, le};
    if (!tok.next(tb, te)) {  // whitespace only
      if (!blank_line) blank_line = line;
      continue;
    }
    if (blank_line) fail(SIVO_EFORMAT, "vocabulary: blank line %d before the node on line %d", blank_line, line);
    int v[34];
    for (int i = 0; i < 34; ++i) {
      if (i > 0 && !tok.next(tb, te)) fail(SIVO_EFORMAT, "vocabulary: line %d has %d of the 34 integer tokens before the weight", line, i);
      if (!parse_int(tb, te, v[i])) fail(SIVO_EFORMAT, "vocabulary: line %d token %d is not an integer", line, i + 1);
    }
    double w;
    if (!tok.next(tb, te)) fail(SIVO_EFORMAT, "vocabulary: line %d has no weight", line);
    if (!parse_double(tb, te, w)) fail(SIVO_EFORMAT, "vocabulary: line %d weight is not a number", line);
    t.parent.push_back(v[0]);
    t.is_leaf.push_back(v[1] > 0 ? 1 : 0);
    for (int i = 0; i < 32; ++i) t.desc.push_back(static_cast<uint8_t>(static_cast<unsigned char>(v[2 + i])));
    t.weight.push_back(w);
  }
  if (t.parent.size() > 2147483647u) fail(SIVO_EFORMAT, "vocabulary: too many nodes");
  check_vocabulary(t.k, t.L, t.scoring, t.weighting, t.parent.data(), t.is_leaf.data(), static_cast<int>(t.parent.size()));
}

Vocabulary::Vocabulary(int dev, int k_, int L_, int scoring_, int weighting_, const int32_t* parent, const uint8_t* is_leaf,
                       const uint8_t* d, const double* weight, int n)
    : device(dev), k(k_), L(L_), scoring(scoring_), weighting(weighting_), n_nodes(n) {
  check_vocabulary(k, L, scoring, weighting, parent, is_leaf, n);
  // children CSR, each parent's children in id order (a counting sort by parent is stable)
  std::vector<int> off(static_cast<size_t>(n) + 1, 0), ch(static_cast<size_t>(n) - 1), word(n, -1);
  for (int i = 1; i < n; ++i) ++off[parent[i] + 1];
  for (int i = 0; i < n; ++i) off[i + 1] += off[i];
  std::vector<int> fill(off.begin(), off.end() - 1);
  for (int i = 1; i < n; ++i) ch[fill[parent[i]]++] = i;
  std::vector<double> ww;
  for (int i = 1; i < n; ++i)
    if (is_leaf[i]) {
      word[i] = static_cast<int>(ww.size());
      ww.push_back(weight[i]);
    }
  n_words = static_cast<int>(ww.size());
  SIVO_CUDA(cudaSetDevice(device));
  desc.alloc(32 * static_cast<size_t>(n));
  child_off.alloc(off.size() * sizeof(int));
  children.alloc(ch.size() * sizeof(int));
  node_word.alloc(word.size() * sizeof(int));
  word_weight.alloc(std::max<size_t>(ww.size(), 1) * sizeof(double));
  SIVO_CUDA(cudaMemcpy(desc.p, d, 32 * static_cast<size_t>(n), cudaMemcpyHostToDevice));
  SIVO_CUDA(cudaMemcpy(child_off.p, off.data(), off.size() * sizeof(int), cudaMemcpyHostToDevice));
  SIVO_CUDA(cudaMemcpy(children.p, ch.data(), ch.size() * sizeof(int), cudaMemcpyHostToDevice));
  SIVO_CUDA(cudaMemcpy(node_word.p, word.data(), word.size() * sizeof(int), cudaMemcpyHostToDevice));
  if (!ww.empty()) SIVO_CUDA(cudaMemcpy(word_weight.p, ww.data(), ww.size() * sizeof(double), cudaMemcpyHostToDevice));
}

}  // namespace sivo
