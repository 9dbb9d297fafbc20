// oracle/ref_rotsum.cpp -- TEST ONLY: the reference's chains that Evaluator::apply_galois_add_inplace and rotate_sum_inplace
// replace, on single seal::Ciphertexts:
//   apply_galois_add: t = encrypted; apply_galois_inplace(t, galois_elt); add_inplace(destination, t)
//   rotate_sum:       for (j = 0; (1 << j) < count; j++) { t = encrypted; rotate_X_inplace(t, step << j); add_inplace(encrypted, t); }
//                     with rotate_X = rotate_vector (CKKS) or rotate_rows (BFV / BGV)
// Compiled into tests/cpp/shim_rotsum_test.cpp by oracle/rotsum.mk.
#include "seal/seal.h"

void ref_apply_galois_add(const seal::Evaluator &ev, seal::Ciphertext &destination, const seal::Ciphertext &encrypted, uint32_t galois_elt,
                          const seal::GaloisKeys &galois_keys)
{
    seal::Ciphertext t = encrypted;
    ev.apply_galois_inplace(t, galois_elt, galois_keys);
    ev.add_inplace(destination, t);
}

void ref_rotate_sum(const seal::Evaluator &ev, bool ckks, seal::Ciphertext &encrypted, int step, size_t count, const seal::GaloisKeys &galois_keys)
{
    for (size_t j = 0; (size_t(1) << j) < count; j++)
    {
        seal::Ciphertext t = encrypted;
        const int s = step * (1 << j);
        if (ckks)
            ev.rotate_vector_inplace(t, s, galois_keys);
        else
            ev.rotate_rows_inplace(t, s, galois_keys);
        ev.add_inplace(encrypted, t);
    }
}
