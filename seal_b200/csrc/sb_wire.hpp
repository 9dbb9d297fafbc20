// seal_b200/csrc/sb_wire.hpp -- the reference's wire format for ciphertexts, host side only (no CUDA):
//   * parms_id = BLAKE2b-256 over [scheme, n, q_0..q_{L-1}, t]            (encryptionparams.cpp:124-158, util/hash.h:30-38)
//   * Ciphertext::save with compr_mode_type::none = SEALHeader + members + DynArray (ciphertext.cpp:190-247,
//     serialization.h:76-91, dynarray.h:662-690)
// so that serialized ciphertexts move between a byte stream and a device slab without a seal::Ciphertext in between
// (SURVEY 8f rank 3).  Seed-compressed members are described here and expanded on the device (sb_prng.cu).
#pragma once
#include "../../include/seal_b200.h"
#include <cstddef>
#include <cstdint>
#include <vector>

namespace sbw
{
    using u64 = unsigned long long;

    // unkeyed BLAKE2b with a 32-byte digest (RFC 7693), digest returned as 4 little-endian words
    void blake2b_256(const void *in, size_t len, u64 out[4]);
    // EncryptionParameters::compute_parms_id for the level with primes q[0..L)
    void parms_id(int scheme, size_t n, const u64 *q, size_t L, u64 t, u64 out[4]);

    constexpr size_t kHeaderBytes = 16;                              // Serialization::SEALHeader
    constexpr size_t kMemberBytes = 32 + 1 + 8 + 8 + 8 + 8 + 8;      // parms_id .. correction_factor
    constexpr size_t kDataOffset = kHeaderBytes + kMemberBytes + kHeaderBytes + 8; // first coefficient word

    // Serialization::Load of a zlib-compressed object (serialization.cpp:236-300, util/ztools.cpp): SEALHeader{compr_mode = zlib,
    // size} followed by ONE zlib stream of the object's body.  Returns false for an uncompressed stream; otherwise fills `plain`
    // with the equivalent uncompressed stream (header with compr_mode none + body) and returns true.  `limit` bounds the
    // decompressed body (the reference bounds loads by the expected in-memory size for the same reason: a malformed stream must
    // not cause arbitrarily large allocations).  zstd streams throw (std::logic_error): the library is not part of this build.
    bool inflate_stream(const uint8_t *p, size_t len, size_t limit, std::vector<uint8_t> &plain);
    // parses and validates one serialized ciphertext (throws std::invalid_argument / std::logic_error like Serialization::Load)
    void inspect(const uint8_t *p, size_t len, sb200_ct_info &info);
    inline size_t save_size(size_t words) { return kDataOffset + 8 * words; }
    // writes everything in front of the coefficient words (kDataOffset bytes) for a ciphertext of info.data_words words
    void write_prefix(const sb200_ct_info &info, uint8_t *out);

    // ---- seed-compressed objects (Serializable<Ciphertext> / <PublicKey> / <RelinKeys> / <GaloisKeys> saved with compr_mode none) ----
    // A seeded ciphertext stream (ciphertext.cpp:190-247, the has_seed_marker branch): the prefix above with a DynArray of the c_0 words
    // only, the words, then UniformRandomGeneratorInfo::save (randomgen.cpp:95-118): its own SEALHeader, prng_type (1 byte), seed (64 bytes).
    constexpr size_t kSeedInfoBytes = kHeaderBytes + 1 + 64;
    inline size_t seeded_save_size(size_t c0_words) { return kDataOffset + 8 * c0_words + kSeedInfoBytes; }
    // writes everything of a seeded stream except the c_0 words (out + kDataOffset .. + 8 info.data_words): info.data_words = L n,
    // info.size = 2; prng = the prng_type c_1 expands with, seed = its 8 words
    void write_seeded(const sb200_ct_info &info, int prng, const u64 seed[8], uint8_t *out);
    // A KSwitchKeys stream (kswitchkeys.cpp:42-86): SEALHeader, parms_id, dim1 = slots, then per slot dim2 and dim2 member streams.
    // `filled` = the indices of the slots that hold `digits` members of member_bytes each, in ascending order; every other slot is a
    // bare dim2 = 0.  RelinKeys: slots 1, filled {0}; GaloisKeys: slots n, filled {(elt - 1) / 2}.
    inline size_t kswitch_save_size(size_t slots, size_t filled, size_t digits, size_t member_bytes)
    {
        return kHeaderBytes + 32 + 8 + 8 * slots + filled * digits * member_bytes;
    }
    // writes the frame (header, parms_id, dim1, every dim2) and returns in first_member[i] the byte offset of the first member of
    // filled[i]; the members of a slot follow one another
    void write_kswitch_frame(const u64 parms_id[4], size_t slots, const std::vector<size_t> &filled, size_t digits, size_t member_bytes,
                             uint8_t *out, std::vector<size_t> &first_member);
    // One entry of a serialized KSwitchKeys object (RelinKeys / GaloisKeys saved with compr_mode_type::none,
    // kswitchkeys.cpp:42-86: SEALHeader, parms_id, dim1, then per slot dim2 and dim2 PublicKey = Ciphertext streams).
    // Returns the byte offsets (from p) of the coefficient words of data()[index][j], j < digits, each 2*L*n words, or L*n words
    // (c_0 only) for a seed-compressed member (KeyGenerator::create_relin_keys / create_galois_keys save their keys so).
    struct KSwitchEntry
    {
        u64 parms_id[4];
        size_t slots = 0;               // data().size()
        size_t L = 0, n = 0;            // shape of every key polynomial pair
        std::vector<size_t> offsets;    // one per decomposition digit
        std::vector<int> seeded;        // per digit: 0, or the prng_type c_1 expands with (1 = blake2xb, 2 = shake256)
        std::vector<size_t> seed_offsets; // per digit: byte offset (from p) of the 64-byte seed of a seeded member, 0 otherwise
    };
    void inspect_kswitch(const uint8_t *p, size_t len, size_t index, KSwitchEntry &entry);
    // Several entries in one pass over the object: entries[i] describes data()[slots[i]].  indices != nullptr: slots = indices[0..count);
    // nullptr: every non-empty slot in slot order (count is ignored).  The frame is parsed up to the last slot needed.  Errors: an index
    // at or past dim1 (std::out_of_range), a duplicated index (std::invalid_argument), a malformed object (std::logic_error), then an
    // empty requested slot (std::invalid_argument, "key not present").  inspect_kswitch is the one-index case.
    void inspect_kswitch_slots(const uint8_t *p, size_t len, const size_t *indices, size_t count, std::vector<size_t> &slots,
                               std::vector<KSwitchEntry> &entries);
} // namespace sbw
