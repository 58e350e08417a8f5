// AudioProcessor.normalize / denormalize (TTS/utils/audio/processor.py:259-337) on one spectrogram value: range
// normalisation (symmetric or not, clipped or not) or the mean-var scaler of a stats_path.  Shared by the vocoder
// hand-off (vocoder_io.cu) and the Griffin-Lim front end (griffin_lim.cu).
#pragma once
#include "../../include/tts_b200.h"

namespace b200tts {

struct NormParams {          // one AudioProcessor's normalisation settings
    int signal_norm, symmetric_norm, clip_norm, has_scaler;
    float max_norm, min_level_db, ref_level_db;
    const float* mean;       // [C] (mean-var scaler) or null
    const float* scale;      // [C]
};

__device__ __forceinline__ float denorm_one(const NormParams& p, float s, int c) {
    if (!p.signal_norm) return s;
    if (p.has_scaler) return __fadd_rn(__fmul_rn(s, p.scale[c]), p.mean[c]);     // StandardScaler.inverse_transform
    if (p.symmetric_norm) {
        if (p.clip_norm) s = fminf(fmaxf(s, -p.max_norm), p.max_norm);
        // ((S + max_norm) * -min_level_db / (2 * max_norm)) + min_level_db   evaluated left to right like numpy
        s = __fadd_rn(__fdiv_rn(__fmul_rn(__fadd_rn(s, p.max_norm), -p.min_level_db), __fmul_rn(2.f, p.max_norm)), p.min_level_db);
        return __fadd_rn(s, p.ref_level_db);
    }
    if (p.clip_norm) s = fminf(fmaxf(s, 0.f), p.max_norm);
    s = __fadd_rn(__fdiv_rn(__fmul_rn(s, -p.min_level_db), p.max_norm), p.min_level_db);
    return __fadd_rn(s, p.ref_level_db);
}

__device__ __forceinline__ float norm_one(const NormParams& p, float s, int c) {
    if (!p.signal_norm) return s;
    if (p.has_scaler) return __fdiv_rn(__fsub_rn(s, p.mean[c]), p.scale[c]);     // StandardScaler.transform
    s = __fsub_rn(s, p.ref_level_db);
    float n = __fdiv_rn(__fsub_rn(s, p.min_level_db), -p.min_level_db);
    if (p.symmetric_norm) {
        n = __fsub_rn(__fmul_rn(__fmul_rn(2.f, p.max_norm), n), p.max_norm);
        if (p.clip_norm) n = fminf(fmaxf(n, -p.max_norm), p.max_norm);
        return n;
    }
    n = __fmul_rn(p.max_norm, n);
    if (p.clip_norm) n = fminf(fmaxf(n, 0.f), p.max_norm);
    return n;
}

inline NormParams to_params(const b200tts_audio_norm& a) {
    NormParams p;
    p.signal_norm = a.signal_norm; p.symmetric_norm = a.symmetric_norm; p.clip_norm = a.clip_norm;
    p.has_scaler = (a.scaler_mean && a.scaler_scale) ? 1 : 0;
    p.max_norm = a.max_norm; p.min_level_db = a.min_level_db; p.ref_level_db = a.ref_level_db;
    p.mean = a.scaler_mean; p.scale = a.scaler_scale;
    return p;
}

}  // namespace b200tts
