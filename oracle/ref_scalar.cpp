// oracle/ref_scalar.cpp -- TEST INFRASTRUCTURE ONLY.
// A flat C wrapper around the UNMODIFIED reference for the tests of the device's scalar CKKS encoder (tests/test_ckks_scalar_oracle.py,
// tests/test_gpu_ckks_scalar.py): a CKKS context (sec_level none, expanded modulus chain) and CKKSEncoder::encode of one double, one
// complex number or one int64 at the level with L primes.  It contains no arithmetic of its own.  Built by oracle/scalar.mk into
// oracle/_ref/libsealref_scalar.so.
#include "seal/seal.h"
#include <complex>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

using namespace seal;

static thread_local std::string g_err;

struct refsc_ctx
{
    std::unique_ptr<SEALContext> context;
    std::unique_ptr<CKKSEncoder> encoder;
    size_t n = 0, k = 0;
};

extern "C" const char *refsc_last_error(void)
{
    return g_err.c_str();
}

extern "C" refsc_ctx *refsc_create(size_t n, const uint64_t *moduli, size_t k)
{
    try
    {
        auto c = std::make_unique<refsc_ctx>();
        EncryptionParameters parms(scheme_type::ckks);
        parms.set_poly_modulus_degree(n);
        parms.set_coeff_modulus(std::vector<Modulus>(moduli, moduli + k));
        c->context = std::make_unique<SEALContext>(parms, true, sec_level_type::none);
        if (!c->context->parameters_set())
            throw std::invalid_argument(c->context->parameter_error_message());
        c->encoder = std::make_unique<CKKSEncoder>(*c->context);
        c->n = n, c->k = k;
        return c.release();
    }
    catch (const std::exception &e)
    {
        g_err = e.what();
        return nullptr;
    }
}

extern "C" void refsc_destroy(refsc_ctx *c)
{
    delete c;
}

// kind 0: encode(double value, parms_id, scale, plain); 1: encode(std::complex<double>{value[0], value[1]}, parms_id, scale, plain);
// 2: encode(std::int64_t value, parms_id, plain).  parms_id: the level with L primes, parms_id_zero for any other L.  out = [L][n]
// words, *out_scale = the plaintext's scale.  Returns 0, 1 on std::invalid_argument (message in refsc_last_error), -1 otherwise.
extern "C" int refsc_ckks_encode_scalar(refsc_ctx *c, size_t L, int kind, const void *value, double scale, uint64_t *out, double *out_scale)
{
    try
    {
        parms_id_type pid = parms_id_zero;
        for (auto cd = c->context->key_context_data(); cd; cd = cd->next_context_data())
            if (cd->parms().coeff_modulus().size() == L)
                pid = cd->parms_id();
        Plaintext p;
        if (kind == 0)
        {
            double v;
            std::memcpy(&v, value, sizeof v);
            c->encoder->encode(v, pid, scale, p);
        }
        else if (kind == 1)
        {
            double v[2];
            std::memcpy(v, value, sizeof v);
            c->encoder->encode(std::complex<double>(v[0], v[1]), pid, scale, p);
        }
        else
        {
            std::int64_t v;
            std::memcpy(&v, value, sizeof v);
            c->encoder->encode(v, pid, p);
        }
        std::memcpy(out, p.data(), L * c->n * sizeof(uint64_t));
        *out_scale = p.scale();
        return 0;
    }
    catch (const std::invalid_argument &e)
    {
        g_err = e.what();
        return 1;
    }
    catch (const std::exception &e)
    {
        g_err = e.what();
        return -1;
    }
}
