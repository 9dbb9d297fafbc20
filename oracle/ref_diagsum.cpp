// oracle/ref_diagsum.cpp -- TEST ONLY: the reference's chains that Evaluator::apply_galois_multiply_plain_add_inplace and
// diagonal_sum replace, on single seal::Ciphertexts:
//   apply_galois_multiply_plain_add: t = encrypted; apply_galois_inplace(t, galois_elt); multiply_plain_inplace(t, plain);
//                                    add_inplace(destination, t)
//   diagonal_sum:                    for each i: t = encrypted; if (steps[i]) rotate_X_inplace(t, steps[i]);
//                                    multiply_plain_inplace(t, diagonals[i]); i == 0 ? destination = t : add_inplace(destination, t)
//                                    with rotate_X = rotate_vector (CKKS) or rotate_rows (BFV / BGV)
// Compiled into tests/cpp/shim_diagsum_test.cpp by oracle/diagsum.mk.
#include "seal/seal.h"
#include <vector>

void ref_apply_galois_multiply_plain_add(const seal::Evaluator &ev, seal::Ciphertext &destination, const seal::Ciphertext &encrypted,
                                         uint32_t galois_elt, const seal::Plaintext &plain, const seal::GaloisKeys &galois_keys)
{
    seal::Ciphertext t = encrypted;
    ev.apply_galois_inplace(t, galois_elt, galois_keys);
    ev.multiply_plain_inplace(t, plain);
    ev.add_inplace(destination, t);
}

void ref_diagonal_sum(const seal::Evaluator &ev, bool ckks, const seal::Ciphertext &encrypted, const std::vector<int> &steps,
                      const std::vector<seal::Plaintext> &diagonals, const seal::GaloisKeys &galois_keys, seal::Ciphertext &destination)
{
    for (size_t i = 0; i < steps.size(); i++)
    {
        seal::Ciphertext t = encrypted;
        if (steps[i])
        {
            if (ckks)
                ev.rotate_vector_inplace(t, steps[i], galois_keys);
            else
                ev.rotate_rows_inplace(t, steps[i], galois_keys);
        }
        ev.multiply_plain_inplace(t, diagonals[i]);
        if (i == 0)
            destination = t;
        else
            ev.add_inplace(destination, t);
    }
}
