// aes_gcm.cuh -- AES-192 (FIPS-197, 12 rounds) and AES-GCM sealing with a 96-bit nonce and a 128-bit tag (NIST SP
// 800-38D) as __host__ __device__ functions, for symmetric_pir.cu's row encryption; tests/emu replays them against
// cryptography's AESGCM.
//
// The round function uses drbg.cuh's tables (make_tables, te0, sub_word): the caller passes the S-box and Te0 it has
// staged.  drbg.cuh's AES-128 functions are not changed.
#pragma once
#include "drbg.cuh"

namespace hecuda {
namespace gcm {

using drbg::u32w;
constexpr int kRounds192 = 12, kRoundKeyWords192 = 4 * (kRounds192 + 1);  // 52

// KeyExpansion (FIPS-197 5.2), 192-bit key as 6 big-endian words: 52 words
HE_HD void expand_key_192(const u32w key[6], u32w *rk, const unsigned char *sbox) {
    for (int i = 0; i < 6; ++i) rk[i] = key[i];
    u32w rcon = 0x01000000u;
    for (int i = 6; i < kRoundKeyWords192; ++i) {
        u32w t = rk[i - 1];
        if (i % 6 == 0) {
            t = drbg::sub_word((t << 8) | (t >> 24), sbox) ^ rcon;
            rcon = (rcon << 1) ^ ((rcon & 0x80000000u) ? 0x1B000000u : 0);
        }
        rk[i] = rk[i - 6] ^ t;
    }
}

// Cipher (FIPS-197 5.1) with `rounds` rounds on the four big-endian columns s[0..3]
HE_HD void encrypt_block(u32w s[4], const u32w *rk, int rounds, const u32w *te0, const unsigned char *sbox) {
    using drbg::ror32;
    u32w a = s[0] ^ rk[0], b = s[1] ^ rk[1], c = s[2] ^ rk[2], d = s[3] ^ rk[3];
    for (int round = 1; round < rounds; ++round) {
        const u32w *k = rk + 4 * round;
        const u32w na = te0[a >> 24] ^ ror32(te0[(b >> 16) & 255], 8) ^ ror32(te0[(c >> 8) & 255], 16) ^ ror32(te0[d & 255], 24) ^ k[0];
        const u32w nb = te0[b >> 24] ^ ror32(te0[(c >> 16) & 255], 8) ^ ror32(te0[(d >> 8) & 255], 16) ^ ror32(te0[a & 255], 24) ^ k[1];
        const u32w nc = te0[c >> 24] ^ ror32(te0[(d >> 16) & 255], 8) ^ ror32(te0[(a >> 8) & 255], 16) ^ ror32(te0[b & 255], 24) ^ k[2];
        const u32w nd = te0[d >> 24] ^ ror32(te0[(a >> 16) & 255], 8) ^ ror32(te0[(b >> 8) & 255], 16) ^ ror32(te0[c & 255], 24) ^ k[3];
        a = na, b = nb, c = nc, d = nd;
    }
    const u32w *k = rk + 4 * rounds;
    s[0] = (((u32w)sbox[a >> 24] << 24) | ((u32w)sbox[(b >> 16) & 255] << 16) | ((u32w)sbox[(c >> 8) & 255] << 8) | sbox[d & 255]) ^ k[0];
    s[1] = (((u32w)sbox[b >> 24] << 24) | ((u32w)sbox[(c >> 16) & 255] << 16) | ((u32w)sbox[(d >> 8) & 255] << 8) | sbox[a & 255]) ^ k[1];
    s[2] = (((u32w)sbox[c >> 24] << 24) | ((u32w)sbox[(d >> 16) & 255] << 16) | ((u32w)sbox[(a >> 8) & 255] << 8) | sbox[b & 255]) ^ k[2];
    s[3] = (((u32w)sbox[d >> 24] << 24) | ((u32w)sbox[(a >> 16) & 255] << 16) | ((u32w)sbox[(b >> 8) & 255] << 8) | sbox[c & 255]) ^ k[3];
}

// X * Y in GCM's GF(2^128) (SP 800-38D 6.3): bit 0 is the most significant bit of hi
HE_HD void gf_mul(u64 &xh, u64 &xl, u64 yh, u64 yl) {
    u64 zh = 0, zl = 0, vh = yh, vl = yl;
    for (int i = 0; i < 128; ++i) {
        const u64 bit = i < 64 ? (xh >> (63 - i)) & 1 : (xl >> (127 - i)) & 1;
        zh ^= vh & (0 - bit), zl ^= vl & (0 - bit);
        const u64 carry = vl & 1;
        vl = (vl >> 1) | (vh << 63);
        vh = (vh >> 1) ^ (0xe100000000000000ull & (0 - carry));
    }
    xh = zh, xl = zl;
}

HE_HD u64 load_be64(const unsigned char *p) {
    u64 v = 0;
    for (int i = 0; i < 8; ++i) v = (v << 8) | p[i];
    return v;
}

// AES.GCM.seal(value, key, nonce) without associated data: out = ciphertext (len bytes) || tag (16 bytes).
// rk: the 52 AES-192 round keys.  Counter blocks are nonce || 32-bit big-endian counter, from J0 + 1 (J0 = nonce || 1).
HE_HD void seal(const u32w *rk, const u32w *te0, const unsigned char *sbox, const unsigned char nonce[12],
                const unsigned char *in, long long len, unsigned char *out) {
    u32w blk[4] = {0, 0, 0, 0};
    encrypt_block(blk, rk, kRounds192, te0, sbox);
    const u64 hh = ((u64)blk[0] << 32) | blk[1], hl = ((u64)blk[2] << 32) | blk[3];  // H = E(0^128)
    const u32w n0 = ((u32w)nonce[0] << 24) | ((u32w)nonce[1] << 16) | ((u32w)nonce[2] << 8) | nonce[3];
    const u32w n1 = ((u32w)nonce[4] << 24) | ((u32w)nonce[5] << 16) | ((u32w)nonce[6] << 8) | nonce[7];
    const u32w n2 = ((u32w)nonce[8] << 24) | ((u32w)nonce[9] << 16) | ((u32w)nonce[10] << 8) | nonce[11];
    u64 sh = 0, sl = 0;  // GHASH state
    u32w counter = 1;
    for (long long at = 0; at < len; at += 16) {
        ++counter;
        u32w ks[4] = {n0, n1, n2, counter};
        encrypt_block(ks, rk, kRounds192, te0, sbox);
        unsigned char c[16];
        const int take = len - at < 16 ? (int)(len - at) : 16;
        for (int j = 0; j < 16; ++j) {
            c[j] = j < take ? (unsigned char)(in[at + j] ^ (ks[j >> 2] >> (24 - 8 * (j & 3)))) : 0;  // zero-padded for GHASH
            if (j < take) out[at + j] = c[j];
        }
        sh ^= load_be64(c), sl ^= load_be64(c + 8);
        gf_mul(sh, sl, hh, hl);
    }
    sl ^= (u64)len * 8;  // the length block: 0 bits of associated data || bits of ciphertext
    gf_mul(sh, sl, hh, hl);
    u32w j0[4] = {n0, n1, n2, 1};
    encrypt_block(j0, rk, kRounds192, te0, sbox);
    for (int j = 0; j < 16; ++j) {
        const u64 s = j < 8 ? sh >> (56 - 8 * j) : sl >> (56 - 8 * (j - 8));
        out[len + j] = (unsigned char)(s ^ (j0[j >> 2] >> (24 - 8 * (j & 3))));
    }
}

// AES.GCM.open(ciphertext || tag, key, nonce) without associated data: in = ciphertext (len bytes), tag = the 16
// received bytes.  The tag is recomputed over the ciphertext and compared with every byte read (no early exit); only
// then is the ciphertext decrypted, with seal's counter blocks, and out gets the plaintext if the tags match and len
// zero bytes if not.  Returns whether they matched.
HE_HD bool open(const u32w *rk, const u32w *te0, const unsigned char *sbox, const unsigned char nonce[12],
                const unsigned char *in, long long len, const unsigned char tag[16], unsigned char *out) {
    u32w blk[4] = {0, 0, 0, 0};
    encrypt_block(blk, rk, kRounds192, te0, sbox);
    const u64 hh = ((u64)blk[0] << 32) | blk[1], hl = ((u64)blk[2] << 32) | blk[3];  // H = E(0^128)
    const u32w n0 = ((u32w)nonce[0] << 24) | ((u32w)nonce[1] << 16) | ((u32w)nonce[2] << 8) | nonce[3];
    const u32w n1 = ((u32w)nonce[4] << 24) | ((u32w)nonce[5] << 16) | ((u32w)nonce[6] << 8) | nonce[7];
    const u32w n2 = ((u32w)nonce[8] << 24) | ((u32w)nonce[9] << 16) | ((u32w)nonce[10] << 8) | nonce[11];
    u64 sh = 0, sl = 0;  // GHASH state
    for (long long at = 0; at < len; at += 16) {
        unsigned char c[16];
        const int take = len - at < 16 ? (int)(len - at) : 16;
        for (int j = 0; j < 16; ++j) c[j] = j < take ? in[at + j] : 0;  // zero-padded
        sh ^= load_be64(c), sl ^= load_be64(c + 8);
        gf_mul(sh, sl, hh, hl);
    }
    sl ^= (u64)len * 8;
    gf_mul(sh, sl, hh, hl);
    u32w j0[4] = {n0, n1, n2, 1};
    encrypt_block(j0, rk, kRounds192, te0, sbox);
    unsigned diff = 0;
    for (int j = 0; j < 16; ++j) {
        const u64 s = j < 8 ? sh >> (56 - 8 * j) : sl >> (56 - 8 * (j - 8));
        diff |= (unsigned char)(s ^ (j0[j >> 2] >> (24 - 8 * (j & 3)))) ^ tag[j];
    }
    const bool ok = diff == 0;
    const unsigned char keep = (unsigned char)(0 - (unsigned)ok);
    u32w counter = 1;
    for (long long at = 0; at < len; at += 16) {
        ++counter;
        u32w ks[4] = {n0, n1, n2, counter};
        encrypt_block(ks, rk, kRounds192, te0, sbox);
        const int take = len - at < 16 ? (int)(len - at) : 16;
        for (int j = 0; j < take; ++j) out[at + j] = (unsigned char)((in[at + j] ^ (ks[j >> 2] >> (24 - 8 * (j & 3)))) & keep);
    }
    return ok;
}

}  // namespace gcm
}  // namespace hecuda
