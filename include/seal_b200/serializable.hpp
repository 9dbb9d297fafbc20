// include/seal_b200/serializable.hpp -- same-signature stand-in for seal::Serializable<T> (native/src/seal/serializable.h): what the
// seal_b200::KeyGenerator and seal_b200::Encryptor overloads without a destination return.
//
//     auto rk = keygen.create_relin_keys();  rk.save(out);             // as with seal::KeyGenerator
//
// It holds the object's uncompressed stream (compr_mode_type::none), written by the device entry points of include/seal_b200.h
// (seeded members: c_0 and the 64-byte seed of c_1).  save with another compression mode passes the members behind the outer
// SEALHeader to the public seal::Serialization::Save, which is how Ciphertext::save and KSwitchKeys::save compress, so the bytes are
// the reference's for every mode its build supports; save_size is the reference's estimate (header + ComprSizeEstimate(members)).
#pragma once

#include "seal/seal.h"
#include <cstddef>
#include <cstdint>
#include <ostream>
#include <utility>
#include <vector>

namespace seal_b200
{
    class KeyGenerator;
    class Encryptor;

    template <class T>
    class Serializable
    {
        friend class KeyGenerator;
        friend class Encryptor;

    public:
        Serializable(const Serializable<T> &copy) = default;
        Serializable(Serializable<T> &&source) = default;
        Serializable &operator=(Serializable<T> &&assign) = default;
        Serializable &operator=(const Serializable<T> &copy) = default;

        // serializable.h: save_size / save(stream) / save(buffer)
        std::streamoff save_size(seal::compr_mode_type compr_mode = seal::Serialization::compr_mode_default) const
        {
            return static_cast<std::streamoff>(kHeader + seal::Serialization::ComprSizeEstimate(stream_.size() - kHeader, compr_mode));
        }
        std::streamoff save(std::ostream &stream, seal::compr_mode_type compr_mode = seal::Serialization::compr_mode_default) const
        {
            return seal::Serialization::Save([this](std::ostream &s) { members(s); }, static_cast<std::streamoff>(stream_.size()), stream,
                                             compr_mode, false);
        }
        std::streamoff save(seal::seal_byte *out, std::size_t size,
                            seal::compr_mode_type compr_mode = seal::Serialization::compr_mode_default) const
        {
            return seal::Serialization::Save([this](std::ostream &s) { members(s); }, static_cast<std::streamoff>(stream_.size()), out, size,
                                             compr_mode, false);
        }

    private:
        static constexpr std::size_t kHeader = sizeof(seal::Serialization::SEALHeader);
        explicit Serializable(std::vector<std::uint8_t> stream) : stream_(std::move(stream))
        {
        }
        // T::save_members: everything behind the outer header
        void members(std::ostream &s) const
        {
            s.write(reinterpret_cast<const char *>(stream_.data() + kHeader), static_cast<std::streamsize>(stream_.size() - kHeader));
        }
        std::vector<std::uint8_t> stream_;
    };
} // namespace seal_b200
