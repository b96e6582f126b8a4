// C ABI entry points of Frame::ComputeBoW: the DBoW2 vocabulary as a device-resident flat tree and
// TemplatedVocabulary::transform(features, BowVector, FeatureVector, levelsup) on it (bow_kernels.cu).
#include <cstring>
#include <memory>
#include <vector>

#include "rgbl_ctx.h"

namespace rgbl {

struct Vocab {
    int device = 0, n_nodes = 0, L = 0;
    DeviceArray<int> child_begin, child_index; DeviceArray<uint8_t> node_desc; DeviceArray<double> node_weight; DeviceArray<int> word_id;
    VocabDev dev() const { return VocabDev{child_begin, child_index, node_desc, node_weight, word_id}; }
};

// descriptors already on the device (desc_dev, n rows)
static int compute_bow_device(Ctx* c, const Vocab* v, int n, const uint8_t* desc_dev, int levelsup, int32_t* bow_word, double* bow_value,
                              int* n_words, int32_t* fv_node, int32_t* fv_start, int32_t* fv_feature, int* n_fv_nodes) {
    TrackBufs& t = c->trk;
    int np2 = 32;
    while (np2 < n) np2 <<= 1;
    // int layout: f_word[n] f_node[n] bow_word[n] fv_node[n] fv_start[n+1] fv_feature[np2] scratch[np2+1] counts[4]
    const size_t ni = (size_t)5 * n + 1 + 2 * (size_t)np2 + 1 + 4;
    if (!t.bw_i.grow(ni, c->scratch_generation) || !t.bw_d.grow((size_t)2 * n + 2, c->scratch_generation)) { c->err = "device allocation failed (BoW scratch)"; return RGBL_E_CUDA; }
    int* f_word = t.bw_i; int* f_node = f_word + n; int* d_bow_word = f_node + n; int* d_fv_node = d_bow_word + n;
    int* d_fv_start = d_fv_node + n; int* d_fv_feature = d_fv_start + n + 1; int* scratch = d_fv_feature + np2; int* counts = scratch + np2 + 1;
    double* f_weight = t.bw_d; double* d_bow_value = f_weight + n;
    stage_begin(c, ST_MATCH, c->st);
    launch_bow_descend(c->st, v->dev(), n, desc_dev, v->L - levelsup, f_word, f_weight, f_node);
    if (launch_bow_assemble(c->st, n, f_word, f_weight, f_node, d_bow_word, d_bow_value, d_fv_node, d_fv_start, d_fv_feature, counts, scratch) < 0) {
        c->err = "too many features for one BoW transform (shared-memory sort holds 8192)"; return RGBL_E_CAPACITY;
    }
    stage_end(c, ST_MATCH, c->st, 2);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(c->h_scalars, counts, 3 * sizeof(int), cudaMemcpyDeviceToHost, c->st));
    CU(cudaStreamSynchronize(c->st));
    const int nw = c->h_scalars[0], nn = c->h_scalars[1], nv = c->h_scalars[2];
    if (nw) {
        CU(cudaMemcpyAsync(bow_word, d_bow_word, (size_t)nw * sizeof(int), cudaMemcpyDeviceToHost, c->st));
        CU(cudaMemcpyAsync(bow_value, d_bow_value, (size_t)nw * sizeof(double), cudaMemcpyDeviceToHost, c->st));
    }
    if (nn) CU(cudaMemcpyAsync(fv_node, d_fv_node, (size_t)nn * sizeof(int), cudaMemcpyDeviceToHost, c->st));
    CU(cudaMemcpyAsync(fv_start, d_fv_start, (size_t)(nn + 1) * sizeof(int), cudaMemcpyDeviceToHost, c->st));
    if (nv) CU(cudaMemcpyAsync(fv_feature, d_fv_feature, (size_t)nv * sizeof(int), cudaMemcpyDeviceToHost, c->st));
    CU(cudaStreamSynchronize(c->st));
    prof_collect(c);
    *n_words = nw; *n_fv_nodes = nn;
    return RGBL_OK;
}

}  // namespace rgbl

using namespace rgbl;

extern "C" {

int rgbl_vocabulary_create(rgbl_ctx* ctx, int n_nodes, const int32_t* child_begin, const int32_t* child_index, const uint8_t* node_desc,
                           const double* node_weight, const int32_t* word_id, int levels, int weighting, int scoring, rgbl_vocabulary** out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!out || n_nodes < 1 || !child_begin || !node_desc || !node_weight || !word_id || levels < 0) { c->err = "bad vocabulary arguments"; return RGBL_E_INVALID; }
    // DBoW2 enums (BowVector.h): WeightingType {TF_IDF, TF, IDF, BINARY}; ScoringType {L1_NORM, L2_NORM, CHI_SQUARE, KL, BHATTACHARYYA, DOT_PRODUCT}
    if (weighting != 0 && weighting != 1) { c->err = "vocabulary weighting IDF / BINARY is not supported (ORBvoc uses TF_IDF)"; return RGBL_E_UNSUPPORTED; }
    if (scoring == 1 || scoring == 5 || scoring < 0 || scoring > 5) { c->err = "vocabulary scoring must normalise with L1 (L1_NORM, CHI_SQUARE, KL, BHATTACHARYYA)"; return RGBL_E_UNSUPPORTED; }
    const int n_child = child_begin[n_nodes];
    if (child_begin[0] != 0 || n_child < 0 || (n_child > 0 && !child_index)) { c->err = "bad vocabulary child table"; return RGBL_E_INVALID; }
    for (int i = 0; i < n_nodes; ++i) if (child_begin[i + 1] < child_begin[i]) { c->err = "vocabulary child_begin is not monotone"; return RGBL_E_INVALID; }
    for (int k = 0; k < n_child; ++k) if (child_index[k] <= 0 || child_index[k] >= n_nodes) { c->err = "vocabulary child index out of range"; return RGBL_E_INVALID; }
    CU(cudaSetDevice(c->cfg.device));
    std::unique_ptr<Vocab> v(new Vocab());
    v->device = c->cfg.device; v->n_nodes = n_nodes; v->L = levels;
    bool ok = v->child_begin.alloc((size_t)n_nodes + 1) == cudaSuccess && v->child_index.alloc(std::max(n_child, 1)) == cudaSuccess &&
              v->node_desc.alloc((size_t)n_nodes * 32) == cudaSuccess && v->node_weight.alloc(n_nodes) == cudaSuccess &&
              v->word_id.alloc(n_nodes) == cudaSuccess;
    ok = ok && cudaMemcpy(v->child_begin, child_begin, (size_t)(n_nodes + 1) * sizeof(int), cudaMemcpyHostToDevice) == cudaSuccess &&
         (n_child == 0 || cudaMemcpy(v->child_index, child_index, (size_t)n_child * sizeof(int), cudaMemcpyHostToDevice) == cudaSuccess) &&
         cudaMemcpy(v->node_desc, node_desc, (size_t)n_nodes * 32, cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(v->node_weight, node_weight, (size_t)n_nodes * sizeof(double), cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(v->word_id, word_id, (size_t)n_nodes * sizeof(int), cudaMemcpyHostToDevice) == cudaSuccess;
    if (!ok) { cudaGetLastError(); c->err = "allocation / upload of the vocabulary failed"; return RGBL_E_CUDA; }
    *out = reinterpret_cast<rgbl_vocabulary*>(v.release());
    return RGBL_OK;
}

void rgbl_vocabulary_destroy(rgbl_vocabulary* voc) {
    Vocab* v = reinterpret_cast<Vocab*>(voc);
    if (!v) return;
    cudaSetDevice(v->device);
    delete v;
}

int rgbl_compute_bow(rgbl_ctx* ctx, const rgbl_vocabulary* voc, int n, const uint8_t* desc, int levelsup, int32_t* bow_word,
                     double* bow_value, int* n_words, int32_t* fv_node, int32_t* fv_start, int32_t* fv_feature, int* n_fv_nodes) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    const Vocab* v = reinterpret_cast<const Vocab*>(voc);
    if (!c) return RGBL_E_INVALID;
    if (c->chain_pending) { c->err = "a tracking chain is in flight (rgbl_resident_track_end not called)"; return RGBL_E_INVALID; }
    if (!v || n < 0 || (n > 0 && !desc) || !n_words || !n_fv_nodes || !fv_start || (n > 0 && (!bow_word || !bow_value || !fv_node || !fv_feature))) {
        c->err = "bad ComputeBoW arguments"; return RGBL_E_INVALID;
    }
    if (v->device != c->cfg.device) { c->err = "vocabulary lives on another device"; return RGBL_E_INVALID; }
    *n_words = 0; *n_fv_nodes = 0; fv_start[0] = 0;
    if (n == 0) return RGBL_OK;
    CU(cudaSetDevice(c->cfg.device));
    TrackBufs& t = c->trk;
    if (!t.q_desc.grow((size_t)n * 32, c->scratch_generation)) { c->err = "device allocation failed (BoW descriptors)"; return RGBL_E_CUDA; }
    CU(cudaMemcpyAsync(t.q_desc, desc, (size_t)n * 32, cudaMemcpyHostToDevice, c->st));
    return compute_bow_device(c, v, n, t.q_desc, levelsup, bow_word, bow_value, n_words, fv_node, fv_start, fv_feature, n_fv_nodes);
}

int rgbl_resident_compute_bow(rgbl_ctx* ctx, const rgbl_vocabulary* voc, int frame, int levelsup, int32_t* bow_word, double* bow_value,
                              int* n_words, int32_t* fv_node, int32_t* fv_start, int32_t* fv_feature, int* n_fv_nodes) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    const Vocab* v = reinterpret_cast<const Vocab*>(voc);
    if (!c) return RGBL_E_INVALID;
    if (c->chain_pending) { c->err = "a tracking chain is in flight (rgbl_resident_track_end not called)"; return RGBL_E_INVALID; }
    if (!v || !n_words || !n_fv_nodes || !fv_start || !bow_word || !bow_value || !fv_node || !fv_feature) { c->err = "bad ComputeBoW arguments"; return RGBL_E_INVALID; }
    if (frame < 0 || frame >= c->last_frames) { c->err = "frame slot out of range"; return RGBL_E_INVALID; }
    if (v->device != c->cfg.device) { c->err = "vocabulary lives on another device"; return RGBL_E_INVALID; }
    CU(cudaSetDevice(c->cfg.device));
    CU(cudaMemcpyAsync(c->h_scalars + 8, c->d_n_sel + frame, sizeof(int), cudaMemcpyDeviceToHost, c->st));
    CU(cudaStreamSynchronize(c->st));
    const int n = c->h_scalars[8];
    *n_words = 0; *n_fv_nodes = 0; fv_start[0] = 0;
    if (n <= 0) return RGBL_OK;
    return compute_bow_device(c, v, n, c->d_desc + (size_t)frame * c->cap_kp * 32, levelsup, bow_word, bow_value, n_words, fv_node, fv_start,
                              fv_feature, n_fv_nodes);
}

}  // extern "C"
