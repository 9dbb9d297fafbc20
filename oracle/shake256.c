/* oracle/shake256.c -- TEST INFRASTRUCTURE ONLY.
 *
 * SHAKE256 written from FIPS 202 (Keccak-f[1600] on lanes A[x + 5y], sponge with a 136-byte rate), and the output stream of the
 * reference's Shake256PRNG (randomgen.cpp:216-227: buffer b = SHAKE256(seed || b as 8 little-endian bytes, 4096 bytes)).  An
 * independent statement for the parity tests of the device's SHAKE256 stream; tests/test_prng_oracle.py pins it against Python's
 * hashlib.shake_256 and against the reference.  Built by oracle/prng.mk into oracle/libshake256.so; the product never loads it.
 */
#include <stddef.h>
#include <stdint.h>
#include <string.h>

static const uint64_t kc_rc[24] = {
    0x0000000000000001ULL, 0x0000000000008082ULL, 0x800000000000808AULL, 0x8000000080008000ULL, 0x000000000000808BULL,
    0x0000000080000001ULL, 0x8000000080008081ULL, 0x8000000000008009ULL, 0x000000000000008AULL, 0x0000000000000088ULL,
    0x0000000080008009ULL, 0x000000008000000AULL, 0x000000008000808BULL, 0x800000000000008BULL, 0x8000000000008089ULL,
    0x8000000000008003ULL, 0x8000000000008002ULL, 0x8000000000000080ULL, 0x000000000000800AULL, 0x800000008000000AULL,
    0x8000000080008081ULL, 0x8000000000008080ULL, 0x0000000080000001ULL, 0x8000000080008008ULL
};
/* rho offsets r[x + 5y] (FIPS 202 table 2) */
static const int kc_rho[25] = { 0, 1, 62, 28, 27, 36, 44, 6, 55, 20, 3, 10, 43, 25, 39, 41, 45, 15, 21, 8, 18, 2, 61, 56, 14 };
static uint64_t kc_rotl(uint64_t v, int s) { return s ? (v << s) | (v >> (64 - s)) : v; }
static void keccak_f1600(uint64_t A[25])
{
    for (int r = 0; r < 24; r++)
    {
        uint64_t C[5], D[5], B[25];
        for (int x = 0; x < 5; x++) /* theta */
            C[x] = A[x] ^ A[x + 5] ^ A[x + 10] ^ A[x + 15] ^ A[x + 20];
        for (int x = 0; x < 5; x++)
            D[x] = C[(x + 4) % 5] ^ kc_rotl(C[(x + 1) % 5], 1);
        for (int y = 0; y < 5; y++) /* rho, pi: (x, y) -> (y, 2x + 3y) */
            for (int x = 0; x < 5; x++)
                B[y + 5 * ((2 * x + 3 * y) % 5)] = kc_rotl(A[x + 5 * y] ^ D[x], kc_rho[x + 5 * y]);
        for (int y = 0; y < 5; y++) /* chi */
            for (int x = 0; x < 5; x++)
                A[x + 5 * y] = B[x + 5 * y] ^ (~B[(x + 1) % 5 + 5 * y] & B[(x + 2) % 5 + 5 * y]);
        A[0] ^= kc_rc[r]; /* iota */
    }
}

/* SHAKE256(in, len bytes) -> out_len bytes; lanes are little-endian, as on the hosts this runs on */
void orc_shake256(const unsigned char *in, size_t len, unsigned char *out, size_t out_len)
{
    enum { RATE = 136 };
    uint64_t A[25] = { 0 };
    unsigned char block[RATE];
    for (;;)
    {
        const size_t take = len < RATE ? len : RATE;
        memset(block, 0, RATE);
        memcpy(block, in, take);
        if (take < RATE) /* the last (possibly empty) block: SHAKE's domain bits 1111, then pad10*1 */
        {
            block[take] ^= 0x1F;
            block[RATE - 1] ^= 0x80;
        }
        for (int i = 0; i < RATE / 8; i++)
        {
            uint64_t lane;
            memcpy(&lane, block + 8 * i, 8);
            A[i] ^= lane;
        }
        keccak_f1600(A);
        in += take, len -= take;
        if (take < RATE)
            break;
    }
    while (out_len)
    {
        const size_t take = out_len < RATE ? out_len : RATE;
        memcpy(out, A, take);
        out += take, out_len -= take;
        if (out_len)
            keccak_f1600(A);
    }
}

/* the first `words` 64-bit words of Shake256PRNG(seed): buffer b = SHAKE256(seed || b, 4096 bytes), b = 0, 1, ... */
void orc_shake256_stream(const uint64_t seed[8], size_t words, uint64_t *out)
{
    uint64_t in[9], buf[512];
    memcpy(in, seed, 64);
    for (size_t w = 0, counter = 0; w < words; counter++)
    {
        in[8] = counter;
        orc_shake256((const unsigned char *)in, sizeof(in), (unsigned char *)buf, sizeof(buf));
        const size_t take = words - w < 512 ? words - w : 512;
        memcpy(out + w, buf, take * 8);
        w += take;
    }
}
