// oracle/ref_multsum.cpp -- TEST ONLY: the reference's chain that sb200_multiply_sum / Evaluator::multiply_sum and
// multiply_relinearize_sum replace, on single seal::Ciphertexts: t_i = lhs[j K + i]; multiply_inplace(t_i, rhs[i]);
// destinations[j] = add_many(t); then, with relin_keys, relinearize_inplace(destinations[j]).
// Compiled into tests/cpp/shim_multsum_test.cpp by oracle/multsum.mk.
#include "seal/seal.h"
#include <vector>

std::vector<seal::Ciphertext> ref_multiply_sum(const seal::Evaluator &ev, const std::vector<seal::Ciphertext> &lhs,
                                               const std::vector<seal::Ciphertext> &rhs, const seal::RelinKeys *relin_keys)
{
    const size_t K = rhs.size(), M = K ? lhs.size() / K : 0;
    std::vector<seal::Ciphertext> out(M);
    for (size_t j = 0; j < M; j++)
    {
        std::vector<seal::Ciphertext> terms;
        for (size_t i = 0; i < K; i++)
        {
            seal::Ciphertext t = lhs[j * K + i];
            ev.multiply_inplace(t, rhs[i]);
            terms.push_back(std::move(t));
        }
        ev.add_many(terms, out[j]);
        if (relin_keys)
            ev.relinearize_inplace(out[j], *relin_keys);
    }
    return out;
}
