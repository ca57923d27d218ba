// The DBoW2 vocabulary (include/sivo_b200.h states the text format and its rules): the host parser and checks (vocabulary.cc), the
// device copy, and the bag-of-words calls on it (bow.cu).
#pragma once
#include <vector>

#include "orb.h"

namespace sivo {

// The tree as sivo_vocabulary_create takes it: one entry per node id, the root at 0.
struct VocTree {
  int k = 0, L = 0, scoring = 0, weighting = 0;
  std::vector<int32_t> parent;
  std::vector<uint8_t> is_leaf;
  std::vector<uint8_t> desc;  // 32 bytes per node
  std::vector<double> weight;
};

// SIVO_ENOENT if unreadable, SIVO_EFORMAT for a malformed file or tree
void parse_vocabulary_text(const char* path, VocTree& t);
// SIVO_EFORMAT for a header or tree the rules refuse
void check_vocabulary(int k, int L, int scoring, int weighting, const int32_t* parent, const uint8_t* is_leaf, int n);

// What the kernels read: children in CSR form (child_off[id] .. child_off[id + 1] in id order), the word of each leaf (-1
// elsewhere) and each word's weight.
struct VocView {
  const uint4* desc;
  const int* child_off;
  const int* children;
  const int* node_word;
  const double* word_weight;
  int L, scoring, weighting;
};

struct Vocabulary {
  int device = 0, k = 0, L = 0, scoring = 0, weighting = 0, n_nodes = 0, n_words = 0;
  DevBuf desc, child_off, children, node_word, word_weight;
  Vocabulary(int device, int k, int L, int scoring, int weighting, const int32_t* parent, const uint8_t* is_leaf, const uint8_t* desc,
             const double* weight, int n);
  VocView view() const {
    return VocView{desc.as<uint4>(), child_off.as<int>(), children.as<int>(), node_word.as<int>(), word_weight.as<double>(), L, scoring,
                   weighting};
  }
};

// ---- bow.cu
void compute_bow_device(const Vocabulary& voc, const Orb& left, const uint8_t* desc, const int* keep_idx, const long long* n_keep,
                        int levelsup, int* node, int* word, int* bow_word, double* bow_weight, long long* bow_len, cudaStream_t s);
void compute_bow_host(const Vocabulary& voc, const uint8_t* desc, int n, int levelsup, int* node, int* word, int* bow_word,
                      double* bow_weight, int* bow_len);
void search_by_bow_device(const Orb& left, const sivo_keypoint* kps, const uint8_t* desc, const int* keep_idx, const long long* n_keep,
                          const int* node, const sivo_keyframe_keys* kfs, const int* const* kf_point, int n_kf, float nnratio, int check,
                          int* match, long long* n_matches, cudaStream_t s);
void search_by_bow_host(const Orb& left, const sivo_keypoint* kps, const uint8_t* desc, const int* node, int n,
                        const sivo_keyframe_keys* kfs, const int* const* kf_point, int n_kf, float nnratio, int check, int* match,
                        long long* n_matches);

}  // namespace sivo
