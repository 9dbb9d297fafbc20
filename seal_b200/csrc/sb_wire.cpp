// seal_b200/csrc/sb_wire.cpp -- see sb_wire.hpp
#include "sb_wire.hpp"
#include <algorithm>
#include <cstring>
#include <stdexcept>
#include <vector>
#include <zlib.h>

namespace sbw
{
    namespace
    {
        constexpr u64 kIv[8] = { 0x6a09e667f3bcc908ull, 0xbb67ae8584caa73bull, 0x3c6ef372fe94f82bull, 0xa54ff53a5f1d36f1ull,
                                 0x510e527fade682d1ull, 0x9b05688c2b3e6c1full, 0x1f83d9abfb41bd6bull, 0x5be0cd19137e2179ull };
        constexpr unsigned char kSigma[10][16] = {
            { 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15 }, { 14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3 },
            { 11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4 }, { 7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8 },
            { 9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13 }, { 2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9 },
            { 12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11 }, { 13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10 },
            { 6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5 }, { 10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0 }
        };
        inline u64 rotr(u64 v, int s) { return (v >> s) | (v << (64 - s)); }
        inline u64 load_le(const unsigned char *p)
        {
            u64 v = 0;
            for (int i = 7; i >= 0; i--)
                v = (v << 8) | p[i];
            return v;
        }

        void compress(u64 h[8], const unsigned char block[128], u64 counter, bool last)
        {
            u64 m[16], v[16];
            for (int i = 0; i < 16; i++)
                m[i] = load_le(block + 8 * i);
            for (int i = 0; i < 8; i++)
                v[i] = h[i], v[i + 8] = kIv[i];
            v[12] ^= counter; // messages here are far below 2^64 bytes: the high counter word stays zero
            if (last)
                v[14] = ~v[14];
            auto mix = [&](int a, int b, int c, int d, u64 x, u64 y) {
                v[a] += v[b] + x, v[d] = rotr(v[d] ^ v[a], 32);
                v[c] += v[d], v[b] = rotr(v[b] ^ v[c], 24);
                v[a] += v[b] + y, v[d] = rotr(v[d] ^ v[a], 16);
                v[c] += v[d], v[b] = rotr(v[b] ^ v[c], 63);
            };
            for (int r = 0; r < 12; r++)
            {
                const unsigned char *s = kSigma[r % 10];
                mix(0, 4, 8, 12, m[s[0]], m[s[1]]);
                mix(1, 5, 9, 13, m[s[2]], m[s[3]]);
                mix(2, 6, 10, 14, m[s[4]], m[s[5]]);
                mix(3, 7, 11, 15, m[s[6]], m[s[7]]);
                mix(0, 5, 10, 15, m[s[8]], m[s[9]]);
                mix(1, 6, 11, 12, m[s[10]], m[s[11]]);
                mix(2, 7, 8, 13, m[s[12]], m[s[13]]);
                mix(3, 4, 9, 14, m[s[14]], m[s[15]]);
            }
            for (int i = 0; i < 8; i++)
                h[i] ^= v[i] ^ v[i + 8];
        }
    } // namespace

    void blake2b_256(const void *in, size_t len, u64 out[4])
    {
        u64 h[8];
        for (int i = 0; i < 8; i++)
            h[i] = kIv[i];
        h[0] ^= 0x01010000ull ^ 32; // parameter block: digest length 32, no key, fanout = depth = 1
        const unsigned char *p = static_cast<const unsigned char *>(in);
        size_t done = 0;
        while (len - done > 128)
        {
            compress(h, p + done, done + 128, false);
            done += 128;
        }
        unsigned char tail[128] = { 0 };
        std::memcpy(tail, p + done, len - done);
        compress(h, tail, len, true);
        for (int i = 0; i < 4; i++)
            out[i] = h[i];
    }

    void parms_id(int scheme, size_t n, const u64 *q, size_t L, u64 t, u64 out[4])
    {
        // [scheme, poly_modulus_degree, coeff_modulus..., plain_modulus] as 64-bit words; a zero plain modulus (CKKS) still
        // occupies one word (Modulus::uint64_count() is 1 for the value 0)
        std::vector<u64> words;
        words.push_back(static_cast<u64>(scheme));
        words.push_back(static_cast<u64>(n));
        words.insert(words.end(), q, q + L);
        words.push_back(t);
        blake2b_256(words.data(), words.size() * sizeof(u64), out);
    }

    namespace
    {
        struct Header
        {
            uint16_t magic;
            uint8_t header_size, major, minor, compr;
            uint16_t reserved;
            uint64_t size;
        };
        static_assert(sizeof(Header) == kHeaderBytes, "SEALHeader is 16 bytes");
        constexpr uint16_t kMagic = 0xA15E;
        constexpr uint8_t kMajor = 4, kMinor = 4; // the reference version this format was restated from (SEAL 4.4.3)

        Header read_header(const uint8_t *p)
        {
            Header h;
            std::memcpy(&h, p, sizeof(h));
            // Serialization::IsCompatibleVersion / IsValidHeader (serialization.h:144-191)
            if (h.major != kMajor || h.minor > kMinor)
                throw std::logic_error("incompatible version");
            if (h.magic != kMagic || h.header_size != kHeaderBytes)
                throw std::logic_error("loaded SEALHeader is invalid");
            if (h.compr != 0)
                throw std::logic_error("unsupported compression mode"); // compressed objects go through inflate_stream first
            if (h.size < kHeaderBytes)
                throw std::logic_error("loaded SEALHeader is invalid");
            return h;
        }
        template <class T>
        T take(const uint8_t *&p)
        {
            T v;
            std::memcpy(&v, p, sizeof(T));
            p += sizeof(T);
            return v;
        }
        template <class T>
        void put(uint8_t *&p, const T &v)
        {
            std::memcpy(p, &v, sizeof(T));
            p += sizeof(T);
        }
    } // namespace

    bool inflate_stream(const uint8_t *p, size_t len, size_t limit, std::vector<uint8_t> &plain)
    {
        if (!p)
            throw std::invalid_argument("in cannot be null");
        if (len < kHeaderBytes)
            throw std::invalid_argument("insufficient size");
        Header h;
        std::memcpy(&h, p, sizeof(h));
        if (h.major != kMajor || h.minor > kMinor)
            throw std::logic_error("incompatible version");
        if (h.magic != kMagic || h.header_size != kHeaderBytes || h.size < kHeaderBytes || h.size > len)
            throw std::logic_error("loaded SEALHeader is invalid");
        if (h.compr == 0)
            return false;
        if (h.compr != 1)
            throw std::logic_error("unsupported compression mode"); // compr_mode_type::zstd: not part of this build
        z_stream z;
        std::memset(&z, 0, sizeof(z));
        if (inflateInit(&z) != Z_OK)
            throw std::logic_error("ZLIB decompression failed");
        plain.assign(kHeaderBytes, 0);
        z.next_in = const_cast<Bytef *>(p + kHeaderBytes);
        size_t in_left = static_cast<size_t>(h.size) - kHeaderBytes;
        std::vector<uint8_t> chunk(size_t(1) << 20);
        int rc = Z_OK;
        while (rc != Z_STREAM_END)
        {
            if (z.avail_in == 0 && in_left)
            {
                const size_t take = std::min<size_t>(in_left, size_t(1) << 30); // uInt is 32 bits wide
                z.avail_in = static_cast<uInt>(take);
                in_left -= take;
            }
            z.next_out = chunk.data();
            z.avail_out = static_cast<uInt>(chunk.size());
            rc = inflate(&z, Z_NO_FLUSH);
            const size_t got = chunk.size() - z.avail_out;
            if ((rc != Z_OK && rc != Z_STREAM_END) || plain.size() - kHeaderBytes + got > limit || (rc == Z_OK && got == 0 && z.avail_in == 0 && !in_left))
            {
                inflateEnd(&z);
                throw std::logic_error("ZLIB decompression failed"); // serialization.cpp:283-289
            }
            plain.insert(plain.end(), chunk.data(), chunk.data() + got);
        }
        inflateEnd(&z);
        h.compr = 0;
        h.size = plain.size();
        std::memcpy(plain.data(), &h, sizeof(h));
        return true;
    }

    void inspect(const uint8_t *p, size_t len, sb200_ct_info &info)
    {
        if (!p)
            throw std::invalid_argument("in cannot be null");
        if (len < kHeaderBytes)
            throw std::invalid_argument("insufficient size");
        const Header outer = read_header(p);
        if (outer.size > len || outer.size < kDataOffset)
            throw std::logic_error("loaded SEALHeader is invalid");
        const uint8_t *r = p + kHeaderBytes;
        std::memset(&info, 0, sizeof(info));
        for (int i = 0; i < 4; i++)
            info.parms_id[i] = take<uint64_t>(r);
        info.is_ntt_form = take<uint8_t>(r) ? 1 : 0;
        info.size = take<uint64_t>(r);
        info.poly_modulus_degree = take<uint64_t>(r);
        info.coeff_modulus_size = take<uint64_t>(r);
        info.scale = take<double>(r);
        info.correction_factor = take<uint64_t>(r);
        // ciphertext.cpp:299-302 checks the metadata against the context; the context-free part of that check is here
        const uint64_t n = info.poly_modulus_degree, L = info.coeff_modulus_size;
        if (info.size < 2 || info.size > 16 || n < 2 || n > 131072 || (n & (n - 1)) || L < 1 || L > 256)
            throw std::logic_error("ciphertext data is invalid");
        const Header inner = read_header(r);
        r += kHeaderBytes;
        const uint64_t count = take<uint64_t>(r);
        if (inner.size != kHeaderBytes + 8 + 8 * count || kHeaderBytes + kMemberBytes + inner.size > outer.size)
            throw std::logic_error("loaded data is invalid");
        if (count == info.size * n * L)
            info.seeded = 0;
        else if (count == n * L && info.size == 2)
            info.seeded = 1; // c_1 is carried as a PRNG seed after the array (ciphertext.cpp:325-352)
        else
            throw std::logic_error("ciphertext data is invalid");
        if (!info.seeded && kHeaderBytes + kMemberBytes + inner.size != outer.size)
            throw std::logic_error("loaded data is invalid");
        if (info.seeded)
        {
            // UniformRandomGeneratorInfo::save behind its own SEALHeader: prng_type (1 byte) + prng_seed_type (64 bytes)
            // (randomgen.cpp:95-118, ciphertext.cpp:334-338)
            const uint8_t *g = r + 8 * count;
            if (kHeaderBytes + kMemberBytes + inner.size + kHeaderBytes + 1 + 64 != outer.size)
                throw std::logic_error("loaded data is invalid");
            const Header ph = read_header(g);
            if (ph.size != kHeaderBytes + 1 + 64)
                throw std::logic_error("loaded data is invalid");
            const uint8_t type = g[kHeaderBytes];
            if (type != 1 && type != 2)
                throw std::logic_error("prng_type is invalid"); // randomgen.cpp:132-136
            info.seeded = type;
            info.seed_offset = static_cast<uint64_t>(g + kHeaderBytes + 1 - p);
        }
        info.data_offset = kDataOffset;
        info.data_words = count;
        info.stream_bytes = outer.size;
    }

    namespace
    {
        // the prefix of a ciphertext stream of `object_bytes` bytes in all (SEALHeader::size)
        void write_prefix_sized(const sb200_ct_info &info, uint8_t *out, size_t object_bytes);
    }
    void write_prefix(const sb200_ct_info &info, uint8_t *out)
    {
        write_prefix_sized(info, out, save_size(info.data_words));
    }

    void write_seeded(const sb200_ct_info &info, int prng, const u64 seed[8], uint8_t *out)
    {
        write_prefix_sized(info, out, seeded_save_size(info.data_words));
        uint8_t *w = out + kDataOffset + 8 * info.data_words;
        const Header h{ kMagic, static_cast<uint8_t>(kHeaderBytes), kMajor, kMinor, 0, 0, kSeedInfoBytes };
        put(w, h);
        put<uint8_t>(w, static_cast<uint8_t>(prng));
        std::memcpy(w, seed, 64);
    }

    void write_kswitch_frame(const u64 parms_id[4], size_t slots, const std::vector<size_t> &filled, size_t digits, size_t member_bytes,
                             uint8_t *out, std::vector<size_t> &first_member)
    {
        uint8_t *w = out;
        const Header h{ kMagic, static_cast<uint8_t>(kHeaderBytes), kMajor, kMinor, 0, 0,
                        kswitch_save_size(slots, filled.size(), digits, member_bytes) };
        put(w, h);
        for (int i = 0; i < 4; i++)
            put<uint64_t>(w, parms_id[i]);
        put<uint64_t>(w, slots);
        first_member.assign(filled.size(), 0);
        for (size_t slot = 0, f = 0; slot < slots; slot++)
        {
            const bool full = f < filled.size() && filled[f] == slot;
            put<uint64_t>(w, full ? digits : 0);
            if (full)
            {
                first_member[f++] = static_cast<size_t>(w - out);
                w += digits * member_bytes;
            }
        }
    }

    namespace
    {
    void write_prefix_sized(const sb200_ct_info &info, uint8_t *out, size_t object_bytes)
    {
        uint8_t *w = out;
        Header h{ kMagic, static_cast<uint8_t>(kHeaderBytes), kMajor, kMinor, 0, 0, object_bytes };
        put(w, h);
        for (int i = 0; i < 4; i++)
            put<uint64_t>(w, info.parms_id[i]);
        put<uint8_t>(w, info.is_ntt_form ? 1 : 0);
        put<uint64_t>(w, info.size);
        put<uint64_t>(w, info.poly_modulus_degree);
        put<uint64_t>(w, info.coeff_modulus_size);
        put<double>(w, info.scale);
        put<uint64_t>(w, info.correction_factor);
        h.size = kHeaderBytes + 8 + 8 * info.data_words;
        put(w, h);
        put<uint64_t>(w, info.data_words);
    }
    } // namespace
    void inspect_kswitch_slots(const uint8_t *p, size_t len, const size_t *indices, size_t count, std::vector<size_t> &slots,
                               std::vector<KSwitchEntry> &entries)
    {
        if (!p)
            throw std::invalid_argument("in cannot be null");
        if (len < kHeaderBytes)
            throw std::invalid_argument("insufficient size");
        const Header outer = read_header(p);
        if (outer.size > len || outer.size < kHeaderBytes + 32 + 8)
            throw std::logic_error("loaded SEALHeader is invalid");
        const uint8_t *r = p + kHeaderBytes, *end = p + outer.size;
        u64 pid[4];
        for (int i = 0; i < 4; i++)
            pid[i] = take<uint64_t>(r);
        const uint64_t dim1 = take<uint64_t>(r);
        if (dim1 > 131072)
            throw std::logic_error("KSwitchKeys outer dimension is invalid"); // kswitchkeys.cpp:121-125
        slots.clear();
        entries.clear();
        // want[slot] = 1 + the slot's position in `indices`, 0 = not requested; the frame is parsed up to the last slot needed
        std::vector<size_t> want;
        uint64_t last = dim1;
        if (indices)
        {
            for (size_t i = 0; i < count; i++)
                if (indices[i] >= dim1)
                    throw std::out_of_range("kswitch_keys_index");
            want.assign(static_cast<size_t>(dim1), 0);
            last = 0;
            for (size_t i = 0; i < count; i++)
            {
                if (want[indices[i]])
                    throw std::invalid_argument("kswitch_keys_index is duplicated");
                want[indices[i]] = i + 1;
                last = std::max<uint64_t>(last, indices[i] + 1);
            }
            slots.assign(indices, indices + count);
            entries.resize(count);
        }
        for (uint64_t slot = 0; slot < last; slot++)
        {
            if (static_cast<size_t>(end - r) < 8)
                throw std::logic_error("loaded data is invalid");
            const uint64_t dim2 = take<uint64_t>(r);
            if (dim2 > 256)
                throw std::logic_error("KSwitchKeys inner dimension is invalid");
            if (!indices && dim2)
            {
                slots.push_back(static_cast<size_t>(slot));
                entries.emplace_back();
            }
            KSwitchEntry *entry = indices ? (want[slot] ? &entries[want[slot] - 1] : nullptr) : (dim2 ? &entries.back() : nullptr);
            if (entry)
            {
                std::memcpy(entry->parms_id, pid, sizeof(pid));
                entry->slots = static_cast<size_t>(dim1);
            }
            for (uint64_t j = 0; j < dim2; j++)
            {
                sb200_ct_info info;
                inspect(r, static_cast<size_t>(end - r), info);
                if (entry)
                {
                    if (info.size != 2 || !info.is_ntt_form || std::memcmp(info.parms_id, pid, sizeof(pid)) != 0 ||
                        (j > 0 && (info.coeff_modulus_size != entry->L || info.poly_modulus_degree != entry->n)))
                        throw std::logic_error("key data is invalid");
                    entry->L = static_cast<size_t>(info.coeff_modulus_size), entry->n = static_cast<size_t>(info.poly_modulus_degree);
                    entry->offsets.push_back(static_cast<size_t>(r - p) + static_cast<size_t>(info.data_offset));
                    entry->seeded.push_back(info.seeded);
                    entry->seed_offsets.push_back(info.seeded ? static_cast<size_t>(r - p) + static_cast<size_t>(info.seed_offset) : 0);
                }
                r += info.stream_bytes;
            }
        }
        for (const KSwitchEntry &e : entries)
            if (e.offsets.empty())
                throw std::invalid_argument("key not present"); // an empty slot (relinkeys.h:84-95, galoiskeys.h:75-86)
    }

    void inspect_kswitch(const uint8_t *p, size_t len, size_t index, KSwitchEntry &entry)
    {
        std::vector<size_t> slots;
        std::vector<KSwitchEntry> entries;
        inspect_kswitch_slots(p, len, &index, 1, slots, entries);
        entry = std::move(entries[0]);
    }
} // namespace sbw
