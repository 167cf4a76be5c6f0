// Fiat–Shamir transcript of the prover and the verifiers: Keccak-256 "SolidityTranscript".
//
// Replaces the `SolidityTranscript` type parameter of
// `PlonkKzgSnark::prove_with_link_hint::<_, _, SolidityTranscript>`
// (/root/reference/crates/circuits/circuit-types/src/traits.rs:996) and of `link_proofs`
// (circuits-core/src/zk_circuits/proof_linking/intent_only.rs:42-47).  The type itself lives in
// the un-vendored mpc-jellyfish fork (plonk/src/transcript/solidity.rs @311568a4); the byte layout
// below is the published jellyfish 0.4 layout as recalled (SURVEY.md App. A) and is kept in this
// one header so it can be aligned with the fork's source when that is available:
//   * append-only byte buffer + 64-byte state;
//   * field elements / curve coordinates appended as 32-byte big-endian canonical integers;
//   * challenge = from_be_bytes_mod_order(state'[..48]),
//     state' = keccak256(state || transcript || 0x00) || keccak256(state || transcript || 0x01).
// Host and device (FF_HD): the prover runs it serially on the host between device rounds, the batch verifier
// (verify_batch.cu) runs one transcript per proof in a device thread.  The byte buffer is a policy: a growing
// std::vector on the host (HostBytes), a caller-sized span of device memory in a kernel (SpanBytes).
#pragma once
#include <cstdint>
#include <cstring>
#include <vector>

#include "ec.cuh"
#include "ff.cuh"

namespace b200 {

// Keccak-256 (pre-FIPS padding, as Ethereum's keccak256), absorbed as a stream: the transcript hashes
// state || buffer || suffix without concatenating them.
class Keccak256 {
  public:
    static constexpr int kRate = 136;
    FF_HD Keccak256() {
        for (auto& v : st_) v = 0;
        pos_ = 0;
    }
    FF_HD void absorb(const uint8_t* data, size_t len) {
        while (len) {  // XOR into the lanes (whole lanes when aligned): the state needs no separate block buffer
            if ((pos_ & 7) == 0 && len >= 8) {
                uint64_t lane = 0;
                for (int b = 0; b < 8; ++b) lane |= (uint64_t)data[b] << (8 * b);
                st_[pos_ >> 3] ^= lane;
                data += 8;
                len -= 8;
                pos_ += 8;
            } else {
                st_[pos_ >> 3] ^= (uint64_t)*data++ << (8 * (pos_ & 7));
                --len;
                ++pos_;
            }
            if (pos_ == kRate) {
                permute(st_);
                pos_ = 0;
            }
        }
    }
    FF_HD void absorb_byte(uint8_t b) { absorb(&b, 1); }
    FF_HD void finish(uint8_t out[32]) {
        st_[pos_ >> 3] ^= (uint64_t)0x01 << (8 * (pos_ & 7));
        st_[(kRate - 1) >> 3] ^= (uint64_t)0x80 << (8 * ((kRate - 1) & 7));
        permute(st_);
        for (int i = 0; i < 32; ++i) out[i] = (uint8_t)(st_[i >> 3] >> (8 * (i & 7)));
    }
    static FF_HD void hash(const uint8_t* data, size_t len, uint8_t out[32]) {
        Keccak256 k;
        k.absorb(data, len);
        k.finish(out);
    }

  private:
    static FF_HD uint64_t rotl(uint64_t x, int s) { return s ? (x << s) | (x >> (64 - s)) : x; }
    static FF_HD void permute(uint64_t a[25]) {
        static const uint64_t round_constants[24] = {
            0x0000000000000001ULL, 0x0000000000008082ULL, 0x800000000000808aULL, 0x8000000080008000ULL,
            0x000000000000808bULL, 0x0000000080000001ULL, 0x8000000080008081ULL, 0x8000000000008009ULL,
            0x000000000000008aULL, 0x0000000000000088ULL, 0x0000000080008009ULL, 0x000000008000000aULL,
            0x000000008000808bULL, 0x800000000000008bULL, 0x8000000000008089ULL, 0x8000000000008003ULL,
            0x8000000000008002ULL, 0x8000000000000080ULL, 0x000000000000800aULL, 0x800000008000000aULL,
            0x8000000080008081ULL, 0x8000000000008080ULL, 0x0000000080000001ULL, 0x8000000080008008ULL};
        // lane (x, y) lives at a[x + 5y]; walk the pi permutation in place with the rho offsets
        constexpr int pi_lane[24] = {10, 7, 11, 17, 18, 3, 5, 16, 8, 21, 24, 4, 15, 23, 19, 13, 12, 2, 20, 14, 22, 9, 6, 1};
        constexpr int rho_off[24] = {1, 3, 6, 10, 15, 21, 28, 36, 45, 55, 2, 14, 27, 41, 56, 8, 25, 43, 62, 18, 39, 61, 20, 44};
#pragma unroll 1
        for (int r = 0; r < 24; ++r) {
            uint64_t col[5];
#pragma unroll
            for (int x = 0; x < 5; ++x) col[x] = a[x] ^ a[x + 5] ^ a[x + 10] ^ a[x + 15] ^ a[x + 20];
#pragma unroll
            for (int x = 0; x < 5; ++x) {
                const uint64_t d = col[(x + 4) % 5] ^ rotl(col[(x + 1) % 5], 1);
#pragma unroll
                for (int y = 0; y < 25; y += 5) a[x + y] ^= d;
            }
            uint64_t carry = a[1];
#pragma unroll
            for (int i = 0; i < 24; ++i) {
                const int j = pi_lane[i];
                const uint64_t tmp = a[j];
                a[j] = rotl(carry, rho_off[i]);
                carry = tmp;
            }
#pragma unroll
            for (int y = 0; y < 25; y += 5) {
                uint64_t row[5];
#pragma unroll
                for (int x = 0; x < 5; ++x) row[x] = a[y + x];
#pragma unroll
                for (int x = 0; x < 5; ++x) a[y + x] = row[x] ^ (~row[(x + 1) % 5] & row[(x + 2) % 5]);
            }
            a[0] ^= round_constants[r];
        }
    }
    uint64_t st_[25];
    int pos_;
};

// Transcript byte buffers.  Host: grows as needed.
struct HostBytes {
    std::vector<uint8_t> v;
    HostBytes() {}
    void append(const uint8_t* p, size_t n) { v.insert(v.end(), p, p + n); }
    const uint8_t* data() const { return v.data(); }
    size_t size() const { return v.size(); }
};
// Device (or host): `cap` bytes owned by the caller, sized for the whole transcript of the item; appends past the
// end are dropped and flagged (`overflow`), so a mis-sized buffer shows up as a failed item, not a stray write.
struct SpanBytes {
    uint8_t* p;
    size_t n, cap;
    bool overflow;
    FF_HD void append(const uint8_t* src, size_t len) {
        if (n + len > cap) {
            overflow = true;
            return;
        }
        for (size_t i = 0; i < len; ++i) p[n + i] = src[i];
        n += len;
    }
    FF_HD const uint8_t* data() const { return p; }
    FF_HD size_t size() const { return n; }
};

template <class Bytes>
class SolidityTranscriptT {
  public:
#pragma nv_exec_check_disable
    FF_HD SolidityTranscriptT() : buf_() {
        for (auto& v : state_) v = 0;
    }
    FF_HD explicit SolidityTranscriptT(const Bytes& b) : buf_(b) {
        for (auto& v : state_) v = 0;
    }

#pragma nv_exec_check_disable
    FF_HD void append_message(const uint8_t* p, size_t n) { buf_.append(p, n); }
    FF_HD void append_u32_be(uint32_t v) {
        const uint8_t b[4] = {(uint8_t)(v >> 24), (uint8_t)(v >> 16), (uint8_t)(v >> 8), (uint8_t)v};
        append_message(b, 4);
    }
    FF_HD void append_u64_be(uint64_t v) {
        uint8_t b[8];
        for (int i = 0; i < 8; ++i) b[i] = (uint8_t)(v >> (56 - 8 * i));
        append_message(b, 8);
    }
    // Montgomery Fr element -> 32 bytes big-endian canonical
    FF_HD void append_field_elem(const fe& a_mont) {
        uint8_t b[32];
        to_be(fe_from_mont<FrCfg>(a_mont), b);
        append_message(b, 32);
    }
    // affine commitment (Montgomery Fq coordinates); the identity is 64 zero bytes
    FF_HD void append_commitment(const g1_affine& c) {
        uint8_t b[32];
        to_be(fe_from_mont<FqCfg>(c.x), b);
        append_message(b, 32);
        to_be(fe_from_mont<FqCfg>(c.y), b);
        append_message(b, 32);
    }
    // get_and_append_challenge: returns the challenge in Montgomery form
#pragma nv_exec_check_disable
    FF_HD fe get_and_append_challenge() {
        Keccak256 k0;  // state || transcript, then the two one-byte suffixes on copies of the sponge
        k0.absorb(state_, 64);
        k0.absorb(buf_.data(), buf_.size());
        Keccak256 k1 = k0;
        k0.absorb_byte(0);
        k1.absorb_byte(1);
        k0.finish(state_);
        k1.finish(state_ + 32);
        // big-endian 48-byte integer mod r, by Horner in Montgomery form
        fe acc = fe_zero();
        const fe c256 = fe_from_u32<FrCfg>(256);
        for (int i = 0; i < 48; ++i) acc = fe_add<FrCfg>(fe_mul<FrCfg>(acc, c256), fe_from_u32<FrCfg>(state_[i]));
        return acc;
    }
    // the 64-byte state after the last challenge (the batch verifier's per-item digest starts from it)
    FF_HD const uint8_t* state() const { return state_; }
    FF_HD const Bytes& bytes() const { return buf_; }

  private:
    static FF_HD void to_be(const fe& canon, uint8_t out[32]) {
        for (int i = 0; i < 8; ++i)
            for (int j = 0; j < 4; ++j) out[31 - (4 * i + j)] = (uint8_t)(canon.l[i] >> (8 * j));
    }
    Bytes buf_;
    uint8_t state_[64];
};

using SolidityTranscript = SolidityTranscriptT<HostBytes>;

}  // namespace b200
