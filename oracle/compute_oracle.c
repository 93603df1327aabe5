/* compute_oracle.c — C restatement of the SM compute probe's operands and answers (include/croprobe.h, "SM compute").
 *
 * Test infrastructure, kept beside the checker (cro_oracle.c) and built the same way into oracle/libcompute_oracle.so;
 * nothing under the package links it.  Written from the header's text, not from csrc/compute.cpp:
 *   element e of call seed `seed` is byte (e mod 8) of pattern_word(seed, e / 8), with e = m * 256 + k for A[m][k] and
 *   e = 32768 + k * 256 + n for B[k][n]; the s8 operand is that byte as int8_t, the small-int operand (byte & 7) - 4;
 *   the answer is D[m][n] = sum over k of A[m][k] * B[k][n].
 */
#include <stdint.h>

#define M 128
#define N 256
#define K 256

static uint64_t splitmix_step(uint64_t seed, uint64_t i) {
    uint64_t z = seed + i + 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

/* Operand element e (0 <= e < M*K + K*N) as answer `answer` reads it: 0 = s8, 1 = small-int. */
int oracle_compute_operand(int answer, uint64_t seed, uint32_t e) {
    const unsigned byte = (unsigned)(splitmix_step(seed, e / 8) >> (8 * (e % 8))) & 0xFFu;
    return answer == 0 ? (int)(int8_t)byte : (int)(byte & 7u) - 4;
}

/* out[m * N + n] = D[m][n], accumulated in 64 bits; returns 0, or -1 for an unknown answer. */
int oracle_compute_answer(int answer, uint64_t seed, int32_t *out) {
    if (answer != 0 && answer != 1) return -1;
    for (int m = 0; m < M; ++m)
        for (int n = 0; n < N; ++n) {
            int64_t d = 0;
            for (int k = 0; k < K; ++k)
                d += (int64_t)oracle_compute_operand(answer, seed, (uint32_t)(m * K + k)) *
                     oracle_compute_operand(answer, seed, (uint32_t)(M * K + k * N + n));
            out[m * N + n] = (int32_t)d;
        }
    return 0;
}
