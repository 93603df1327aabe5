// compute.hpp — host side of the SM compute probe (cro_probe_compute): the operands and the expected answers.
#pragma once
#include <stdint.h>

#include "../../include/croprobe.h"

namespace cro {
namespace compute {

constexpr int kTile = CRO_COMPUTE_M * CRO_COMPUTE_N;

// The answer tile of the operands of `seed` (include/croprobe.h): answer CRO_COMPUTE_ANSWER_S8 or _SMALL, M x N int32
// values, row-major.  CRO_ERR_INVALID_ARG for another answer.
int Expected(int answer, uint64_t seed, int32_t* out);

// sum over the 256 threads of a CTA of sum_j tile[row(t, j)][col(t, j)] * (2j + 1) (mod 2^64): what one iteration adds
// to a CTA's running fold when every value is right.
uint64_t CtaFold(const int32_t* tile);

}  // namespace compute
}  // namespace cro
