// Bag-of-words assembly ORACLE — TEST INFRASTRUCTURE ONLY.
//
// The bookkeeping half of DBoW2's TemplatedVocabulary::transform(features, v, fv, levelsup)
// (reference Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1150-1216) with TF_IDF weighting and L1 normalisation (the
// ORBvoc settings), restated over ordered maps from the per-feature (word id, weight, node id) triples that
// voc_oracle_transform (oracle/bow_oracle.cpp) returns:
//   * a feature takes part only when its weight is > 0 (:1181);
//   * BowVector::addWeight (BowVector.cpp): the first feature of a word inserts its weight, each later one adds to it;
//   * FeatureVector::addFeature (FeatureVector.cpp): the feature index is appended to its node's list;
//   * BowVector::normalize(L1) (BowVector.cpp:62-84): the norm is the sum of |value| in map (ascending word) order, and
//     every value is divided by it when it is > 0.
// Node id -1 (the leaf is shallower than the requested level; the reference leaves the id unset) is kept as a signed key,
// so it sorts first. Pinned by an independent Python restatement in tests/test_bow_assembly_oracle.py; only tests/ and
// tools/ load this.
#include <cmath>
#include <map>
#include <vector>

extern "C" {

// n features -> BowVector (bow_word / bow_value [n], *n_words) and FeatureVector (fv_node [n], fv_ptr [n+1], fv_feat [n],
// *n_node), each in ascending key order
__attribute__((visibility("default"))) void bow_oracle_assemble(const int* word, const double* weight, const int* node, int n,
                                                                int* bow_word, double* bow_value, int* n_words, int* fv_node,
                                                                int* fv_ptr, int* fv_feat, int* n_node) {
    std::map<int, double> v;
    std::map<int, std::vector<int>> fv;
    for (int i = 0; i < n; ++i) {
        if (!(weight[i] > 0)) continue;
        const auto it = v.find(word[i]);
        if (it != v.end()) it->second += weight[i];
        else v.emplace(word[i], weight[i]);
        fv[node[i]].push_back(i);
    }
    double norm = 0.0;
    for (const auto& kv : v) norm += std::fabs(kv.second);
    if (norm > 0.0)
        for (auto& kv : v) kv.second /= norm;
    int k = 0;
    for (const auto& kv : v) { bow_word[k] = kv.first; bow_value[k] = kv.second; ++k; }
    *n_words = k;
    int nd = 0, f = 0;
    fv_ptr[0] = 0;
    for (const auto& kv : fv) {
        fv_node[nd] = kv.first;
        for (const int i : kv.second) fv_feat[f++] = i;
        fv_ptr[++nd] = f;
    }
    *n_node = nd;
}

}  // extern "C"
