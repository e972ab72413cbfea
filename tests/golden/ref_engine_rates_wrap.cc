// TEST INFRASTRUCTURE ONLY, used by make_golden_fbank_rates.py (never built into the package): a C entry point over the
// UNMODIFIED reference class wespeaker::SpeakerEngine (runtime/core/speaker/speaker_engine.cc:30-139) at any
// (sample_rate, feat_dim), as `SpeakerEngine(model, feat_dim, sample_rate, ...)` is constructed by the reference runtime.
// The generator compiles this file together with the reference's speaker_engine.cc, feature_pipeline.cc and fft.cc from a
// wespeaker checkout and oracle/ref_shim/glog, the same sources oracle/Makefile compiles for libref_engine.so.
// Every standard header the reference headers pull in is included BEFORE the access hack below.
#include <algorithm>
#include <cmath>
#include <condition_variable>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <functional>
#include <iostream>
#include <limits>
#include <map>
#include <memory>
#include <mutex>
#include <numeric>
#include <queue>
#include <random>
#include <sstream>
#include <string>
#include <thread>
#include <unordered_map>
#include <utility>
#include <vector>

#include "glog/logging.h"

#define private public   // ApplyMean is private in the reference header; the wrapper only calls it
#include "speaker/speaker_engine.h"
#undef private

extern "C" {

// SpeakerEngine("", feat_dim, sample_rate, 256, samples_per_chunk).ExtractFeature(pcm) (+ ApplyMean per chunk when
// apply_mean != 0).  Returns the number of chunks; shape[0..2] = {chunks, frames per chunk, feat_dim}; *out is malloc'ed
// [chunks][frames][dim] floats (free with ref_rates_free).
int ref_extract_feature_at(const short* pcm, int nsamples, int samples_per_chunk, int apply_mean, int sample_rate, int feat_dim,
                           float** out, int* shape) {
    wespeaker::SpeakerEngine eng("", feat_dim, sample_rate, 256, samples_per_chunk);
    std::vector<std::vector<std::vector<float>>> chunks;
    eng.ExtractFeature(pcm, nsamples, &chunks);
    const int nc = (int)chunks.size();
    shape[0] = nc; shape[1] = nc ? (int)chunks[0].size() : 0; shape[2] = (nc && shape[1]) ? (int)chunks[0][0].size() : 0;
    for (auto& c : chunks)
        if ((int)c.size() != shape[1]) return -1;          // ragged chunk lists (full mode has exactly one)
    *out = (float*)malloc(sizeof(float) * (size_t)(nc ? nc : 1) * (shape[1] ? shape[1] : 1) * (shape[2] ? shape[2] : 1));
    float* p = *out;
    for (auto& c : chunks) {
        if (apply_mean) eng.ApplyMean(&c, (unsigned)shape[2]);
        for (auto& row : c) { memcpy(p, row.data(), sizeof(float) * row.size()); p += row.size(); }
    }
    return nc;
}

void ref_rates_free(float* p) { free(p); }

}  // extern "C"
