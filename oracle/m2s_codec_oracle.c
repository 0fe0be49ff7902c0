/* m2s_codec_oracle.c — the per-value encodings of parsers::savePlyVector and decodings of parsers::loadPlyFile, written
 * the way the reference writes them and calling glibc's logf / expf as the reference does (TEST INFRASTRUCTURE: the
 * checker of the device functions in mesh2splat_b200/csrc/m2s_codec.cuh, on every input bit pattern).  Built with gcc
 * -ffp-contract=off and no fast-math: every operation is one IEEE fp32 (or fp64) rounding.  The loops are split over the
 * host's cores (OpenMP); each element is independent, so the result does not depend on the split.
 *
 * Every entry: out[i] = f(in[i]) for i < n. */
#include <math.h>
#include <stdint.h>

#define ORC_API __attribute__((visibility("default")))

static const float kShC0 = 0.28209479177387814f; /* SH_COEFF0, params.hpp:17 */

/* utils::getShFromColor (utils.cpp:47) */
ORC_API void orc_codec_sh0(const float* in, uint64_t n, float* out) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n; ++i) out[i] = (in[i] - 0.5f) / kShC0;
}

/* utils::invSigmoid (utils.hpp:270): std::clamp (NaN passes), then -std::log of a float */
ORC_API void orc_codec_logit(const float* in, uint64_t n, float* out) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n; ++i) {
        float a = in[i];
        a = a < 0.0f ? 0.0f : (1.0f < a ? 1.0f : a);
        out[i] = -logf((1.0f / (a + 1e-8f)) - 1.0f);
    }
}

/* parsers.cpp:497-499: std::log(scale * scaleMultiplier) */
ORC_API void orc_codec_log_scale(const float* in, uint64_t n, float mult, float* out) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n; ++i) out[i] = logf(in[i] * mult);
}

/* glm::exp of a float (parsers.cpp:590-592) */
ORC_API void orc_codec_expf(const float* in, uint64_t n, float* out) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n; ++i) out[i] = expf(in[i]);
}

/* utils::sigmoid (utils.hpp:269): 1.0 / (1.0 + std::exp(-opacity)), the exp in fp32, the rest in fp64 */
ORC_API void orc_codec_sigmoid(const float* in, uint64_t n, float* out) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n; ++i) out[i] = (float)(1.0 / (1.0 + (double)expf(-in[i])));
}
