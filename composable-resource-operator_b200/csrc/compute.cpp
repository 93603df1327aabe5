// compute.cpp — the SM compute probe's expected answers, computed on the host (include/croprobe.h, "SM compute").
//
// Each answer is an exact integer product: |s8 x s8| <= 2^14, so a sum over K = 256 stays within 2^22; |small-int
// products| <= 16, so every partial sum stays within 2^12.  int32 accumulation is exact for both.
#include "compute.hpp"

#include <vector>

#include "kernels.cuh"

namespace cro {
namespace compute {

namespace {
constexpr int M = CRO_COMPUTE_M, N = CRO_COMPUTE_N, K = CRO_COMPUTE_K;

inline int operand_value(int answer, unsigned byte) {
    return answer == CRO_COMPUTE_ANSWER_S8 ? (int)(int8_t)byte : (int)(byte & 7u) - 4;
}
}  // namespace

int Expected(int answer, uint64_t seed, int32_t* out) {
    if ((answer != CRO_COMPUTE_ANSWER_S8 && answer != CRO_COMPUTE_ANSWER_SMALL) || !out) return CRO_ERR_INVALID_ARG;
    static_assert(M * K % 8 == 0 && K * N % 8 == 0, "operands are whole pattern words");
    std::vector<int32_t> a(M * K), b(K * N);        // A[m][k], B[k][n]
    for (uint32_t w = 0; w < (uint32_t)(M * K + K * N) / 8; ++w) {
        const uint64_t v = pattern_word(seed, w);
        for (uint32_t j = 0; j < 8; ++j) {          // element e is byte e % 8 of pattern_word(seed, e / 8)
            const uint32_t e = 8 * w + j;
            const int x = operand_value(answer, (unsigned)(v >> (8 * j)) & 0xFFu);
            if (e < (uint32_t)(M * K)) a[e] = x;
            else b[e - M * K] = x;
        }
    }
    for (int m = 0; m < M; ++m) {
        int32_t row[N] = {};
        for (int k = 0; k < K; ++k) {
            const int32_t x = a[m * K + k];
            const int32_t* bk = b.data() + k * N;
            for (int n = 0; n < N; ++n) row[n] += x * bk[n];
        }
        for (int n = 0; n < N; ++n) out[m * N + n] = row[n];
    }
    return CRO_OK;
}

uint64_t CtaFold(const int32_t* tile) {
    uint64_t f = 0;
    for (unsigned t = 0; t < 256; ++t) {
        const unsigned r0 = 64 * (t / 128) + 16 * ((t / 32) % 4) + (t % 32) / 4, c0 = 2 * (t % 4);
        for (unsigned j = 0; j < 128; ++j) {
            const unsigned row = r0 + 8 * ((j / 2) % 2), col = 8 * (j / 4) + c0 + j % 2;
            f += (uint64_t)(int64_t)tile[row * N + col] * (2 * j + 1);
        }
    }
    return f;
}

}  // namespace compute
}  // namespace cro
