// oracle/ref_plainsum.cpp -- TEST ONLY: the reference's chain that sb200_multiply_plain_sum / Evaluator::multiply_plain_sum replace,
// on single seal::Ciphertexts: t_i = encrypteds[i]; multiply_plain_inplace(t_i, plains[j K + i]); destinations[j] = add_many(t).
// Compiled into tests/cpp/shim_plainsum_test.cpp by oracle/plainsum.mk.
#include "seal/seal.h"
#include <vector>

std::vector<seal::Ciphertext> ref_multiply_plain_sum(const seal::Evaluator &ev, const std::vector<seal::Ciphertext> &encrypteds,
                                                     const std::vector<const seal::Plaintext *> &plains)
{
    const size_t K = encrypteds.size(), M = K ? plains.size() / K : 0;
    std::vector<seal::Ciphertext> out(M);
    for (size_t j = 0; j < M; j++)
    {
        std::vector<seal::Ciphertext> terms;
        for (size_t i = 0; i < K; i++)
        {
            seal::Ciphertext t = encrypteds[i];
            ev.multiply_plain_inplace(t, *plains[j * K + i]);
            terms.push_back(std::move(t));
        }
        ev.add_many(terms, out[j]);
    }
    return out;
}
