// frontend.cpp -- the HOST front half in front of the CUDA synthesis path (include/lewton_frontend.h):
// Vorbis header parsing, audio-packet entropy decode up to the cut at audio.rs:986, Ogg paging and
// the OggStreamReader loop.  Bit-serial CPU work by nature; every function cites the reference code
// whose behaviour (including its quirks) it restates.  f32 arithmetic is written in the reference's
// expression order and compiled without contraction (-ffp-contract=off, csrc/Makefile).
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <memory>
#include <new>
#include <stdexcept>
#include <string>
#include <thread>
#include <utility>
#include <vector>

#include "../../include/lewton_frontend.h"
#include "batcher.h"

// Resource caps for header fields a hostile stream controls (BufferNotAddressable, header.rs:117-125):
// the spec allows 2^24 codebook entries; value tables beyond 2^26 floats are refused.  The fuzz harness
// (tests/fuzz) lowers both so that it spends its time in the parser, not in the allocator.
#ifndef LWF_MAX_ENTRIES
#define LWF_MAX_ENTRIES (1u << 24)
#endif
#ifndef LWF_MAX_VQ_ELEMS
#define LWF_MAX_VQ_ELEMS (1ull << 26)
#endif

namespace lwf {

// ---------------------------------------------------------------------------------------------
// bitpacking.rs: BitpackCursor.  LSB-first; a read succeeds iff all its bits lie inside the buffer
// and leaves the cursor untouched otherwise (bpc_read_body!, bitpacking.rs:93-160); a dynamic read
// of 0 bits is Ok(0) (:283-290).
// ---------------------------------------------------------------------------------------------
struct BitReader {
    const uint8_t *p;
    size_t len;
    size_t pos = 0;        // bit position
    BitReader(const uint8_t *d, size_t n) : p(d), len(n) {}
    size_t bits_left() const { return len * 8 - pos; }
    // the next min(57, bits_left()) bits at least, first bit in bit 0, zero beyond the end of the data
    uint64_t peek() const
    {
        const size_t byte = pos >> 3;
        uint64_t w = 0;
        if (byte + 8 <= len) {
            std::memcpy(&w, p + byte, 8);                   // little endian hosts (x86-64, aarch64)
        } else {
            for (size_t i = byte; i < len; i++) w |= (uint64_t)p[i] << (8 * (i - byte));
        }
        return w >> (pos & 7);
    }
    bool read(unsigned nbits, uint64_t *out)
    {
        if (nbits == 0) { *out = 0; return true; }
        if (pos + nbits > len * 8) return false;
        uint64_t v;
        if (nbits <= 57) {
            v = peek() & (~0ull >> (64 - nbits));
        } else {                                             // up to 64 bits: two pieces
            v = peek() & ((1ull << 32) - 1);
            pos += 32;
            v |= (peek() & (~0ull >> (64 - (nbits - 32)))) << 32;
            pos -= 32;
        }
        pos += nbits;
        *out = v;
        return true;
    }
    bool u(unsigned nbits, uint32_t *out)
    {
        uint64_t v;
        if (!read(nbits, &v)) return false;
        *out = (uint32_t)v;
        return true;
    }
    bool flag(bool *out)
    {
        if (pos >= len * 8) return false;
        *out = (p[pos >> 3] >> (pos & 7)) & 1;
        pos++;
        return true;
    }
};

// lib.rs:166-172
static inline uint8_t ilog(uint64_t val)
{
    uint8_t r = 0;
    while (val) { r++; val >>= 1; }
    return r;
}

// bitpacking.rs:304-314
static inline float float32_unpack(uint32_t val)
{
    const uint32_t sgn = val & 0x80000000u, exp = (val & 0x7fe00000u) >> 21;
    const double mantissa = (double)(val & 0x1fffffu);
    const double signed_mantissa = sgn ? -mantissa : mantissa;
    return (float)signed_mantissa * exp2f((float)exp - 788.0f);
}

// ---------------------------------------------------------------------------------------------
// huffman_tree.rs: VorbisHuffmanTree.  Entries are inserted in order, each at the leftmost free
// position of its depth (HuffTree::insert_rec, :60-108); the flat program (:156-180) is
// [has_children << 31 | payload, left, right] per node.
// ---------------------------------------------------------------------------------------------
enum { HUFF_OK = 0, HUFF_OVERSPECIFIED, HUFF_UNDERPOPULATED, HUFF_INVALID_SINGLE };

struct Huffman {
    static constexpr unsigned kPeek = 10;       // first-level lookup: the next 10 bits -> leaf or inner node
    std::vector<uint32_t> prog;
    std::vector<uint32_t> fast;                 // [1 << kPeek]: (payload << 5) | bits consumed for codewords of <= kPeek bits,
                                                // else 1 << 31 | (node position << 5) | kPeek
    bool single = false;        // one entry of length 1: both bit values decode to it (:131-143)
    uint32_t single_payload = 0;
    bool empty = true;          // no used entry: the reference would index out of bounds on a read

    struct Node { bool even = true; bool has_payload = false; uint32_t payload = 0; int l = -1, r = -1; };

    static bool insert(std::vector<Node> &t, int at, uint32_t payload, unsigned depth)
    {
        if (t[at].has_payload) return false;
        if (depth == 0) {
            if (t[at].l >= 0 || t[at].r >= 0) return false;
            t[at].has_payload = true;
            t[at].payload = payload;
            return true;
        }
        if (t[at].even) {
            if (t[at].l >= 0) return false;
            const int nn = (int)t.size();
            t.push_back(Node());
            insert(t, nn, payload, depth - 1);
            t[at].l = nn;
            t[at].even = false;
            return true;
        }
        const int left = t[at].l;
        if (!t[left].even) {
            if (insert(t, left, payload, depth - 1)) {
                t[at].even = t[left].even && (t[at].r >= 0 ? t[t[at].r].even : false);
                return true;
            }
        }
        if (t[at].r >= 0) {
            const bool ok = insert(t, t[at].r, payload, depth - 1);
            t[at].even = t[left].even && t[t[at].r].even;
            return ok;
        }
        const int nn = (int)t.size();
        t.push_back(Node());
        const bool ok = insert(t, nn, payload, depth - 1);
        t[at].even = t[left].even && t[nn].even;
        t[at].r = nn;
        return ok;
    }

    uint32_t flatten(const std::vector<Node> &t, int at)
    {
        const uint32_t cur = (uint32_t)prog.size();
        const bool kids = t[at].l >= 0 || t[at].r >= 0;
        prog.push_back(((uint32_t)kids << 31) | (t[at].has_payload ? t[at].payload : 0));
        if (kids) {
            prog.push_back(0);
            prog.push_back(0);
            const uint32_t l = flatten(t, t[at].l);
            prog[cur + 1] = l;
            const uint32_t r = flatten(t, t[at].r);
            prog[cur + 2] = r;
        }
        return cur;
    }

    // VorbisHuffmanTree::load_from_array, huffman_tree.rs:113-214
    int load(const std::vector<uint8_t> &lengths)
    {
        std::vector<Node> t(1);
        t.reserve(lengths.size() * 2 + 2);
        size_t cnt = 0, last = 0;
        for (size_t i = 0; i < lengths.size(); i++) {
            if (!lengths[i]) continue;
            cnt++;
            last = i;
            if (!insert(t, 0, (uint32_t)i, lengths[i])) return HUFF_OVERSPECIFIED;
        }
        empty = cnt == 0;
        if (cnt == 1) {
            if (lengths[last] != 1) return HUFF_INVALID_SINGLE;
            single = true;
            single_payload = (uint32_t)last;
            return HUFF_OK;
        }
        if (!t[0].even) return HUFF_UNDERPOPULATED;
        if (!empty) {
            flatten(t, 0);
            // the walk of read() for every 10-bit prefix, done once (the reference unrolls 8 bits, huffman_tree.rs:182-208)
            fast.resize(1u << kPeek);
            // (node positions must fit 26 bits beside the flag and the bit count: a tree of more than ~11 M entries -- legal,
            // never seen -- is walked from the root, bit by bit)
            const bool walk_only = prog.size() >= (1u << 26);
            for (uint32_t bits = 0; bits < (1u << kPeek); bits++) {
                if (walk_only) { fast[bits] = 0x80000000u; continue; }
                uint32_t at = 0, used = 0;
                while (used < kPeek && (prog[at] & 0x80000000u)) {
                    at = prog[at + 1 + ((bits >> used) & 1)];
                    used++;
                }
                // a codeword that ends within the peeked bits: the entry carries the payload itself (one load per
                // symbol instead of two dependent ones); else bit 31 and the node to go on from
                const uint32_t e = prog[at];
                if (e & 0x80000000u) fast[bits] = 0x80000000u | (at << 5) | used;
                else fast[bits] = (e << 5) | used;
            }
        }
        return HUFF_OK;
    }

    // BitpackCursor::read_huffman, bitpacking.rs:455-486 (the 8-bit peek table is a shortcut for the
    // same walk); false = the packet ended inside the codeword, all remaining bits consumed
    bool read(BitReader &rdr, uint32_t *out) const
    {
        if (single) {
            bool b;
            if (!rdr.flag(&b)) return false;
            *out = single_payload;
            return true;
        }
        if (empty) return false;
        // table step: as many of the next 10 bits as the walk needs.  Bits past the end of the packet read
        // as zero; a codeword that would need them fails exactly like the bit-by-bit walk (which consumes
        // what is left and then reports the end of the packet).
        const size_t left = rdr.bits_left();
        const uint32_t f = fast[rdr.peek() & ((1u << kPeek) - 1)];
        const uint32_t used = f & 31;
        if (used > left) { rdr.pos += left; return false; }
        rdr.pos += used;
        if (!(f & 0x80000000u)) { *out = f >> 5; return true; }
        uint32_t at = (f & 0x7fffffffu) >> 5;
        uint32_t e = prog[at];
        while (e & 0x80000000u) {                            // codewords longer than 10 bits: keep walking
            bool b;
            if (!rdr.flag(&b)) return false;
            at = prog[at + 1 + (b ? 1 : 0)];
            e = prog[at];
        }
        *out = e;
        return true;
    }
};

// ---------------------------------------------------------------------------------------------
// header.rs
// ---------------------------------------------------------------------------------------------
struct Codebook {                    // header.rs:360-368
    uint16_t dimensions = 0;
    bool has_vq = false;
    std::vector<float> vq;           // codebook_vq_lookup_vec: [entries][dimensions]
    Huffman tree;
};

struct ResidueBook { uint8_t vals_used = 0; uint8_t val[8] = {0, 0, 0, 0, 0, 0, 0, 0}; };

struct Residue {                     // header.rs:370-379
    uint8_t type = 0;
    uint32_t begin = 0, end = 0, partition_size = 0;
    uint8_t classifications = 0, classbook = 0;
    std::vector<ResidueBook> books;
};

struct Mapping {                     // header.rs:381-388
    std::vector<uint8_t> magnitudes, angles, mux, submap_floors, submap_residues;
};

struct ModeInfo { bool blockflag = false; uint8_t mapping = 0; };

struct Floor0 {                      // header.rs:399-407
    uint8_t order = 0, amplitude_bits = 0, amplitude_offset = 0, number_of_books = 0;
    uint16_t rate = 0, bark_map_size = 0;
    std::vector<uint8_t> book_list;
    std::vector<float> bark_cos_omega[2];
};

struct Floor1 {                      // header.rs:409-419
    uint8_t multiplier = 1;
    std::vector<uint8_t> partition_class, class_dimensions, class_subclasses, class_masterbooks;
    std::vector<std::vector<int16_t>> subclass_books;
    std::vector<uint32_t> x_list;
};

struct Floor { int type = 1; Floor0 f0; Floor1 f1; };

struct Ident {                       // header.rs:188-211
    uint8_t audio_channels = 0, blocksize_0 = 0, blocksize_1 = 0;
    uint32_t audio_sample_rate = 0;
    int32_t bitrate_maximum = 0, bitrate_nominal = 0, bitrate_minimum = 0;
};

struct Headers {
    Ident ident;
    std::string vendor;
    std::vector<std::pair<std::string, std::string>> comments;
    std::vector<Codebook> codebooks;
    std::vector<Floor> floors;
    std::vector<Residue> residues;
    std::vector<Mapping> mappings;
    std::vector<ModeInfo> modes;
};

#define RD(expr) do { if (!(expr)) return LWF_ERR_END_OF_PACKET; } while (0)
#define BAD() return LWF_ERR_HEADER_BAD_FORMAT

// read_header_begin, header.rs:131-155
static int read_header_begin(BitReader &rdr, uint8_t *type)
{
    uint32_t v;
    RD(rdr.u(8, &v));
    if (!(v & 1)) return LWF_ERR_HEADER_IS_AUDIO;
    *type = (uint8_t)v;
    static const uint8_t magic[6] = {0x76, 0x6f, 0x72, 0x62, 0x69, 0x73};
    for (int i = 0; i < 6; i++) {
        uint32_t c;
        RD(rdr.u(8, &c));
        if (c != magic[i]) return LWF_ERR_NOT_VORBIS_HEADER;      // && short-circuits: stop at the first mismatch
    }
    return LWB_OK;
}

// read_header_ident, header.rs:221-259
static int read_ident(const uint8_t *d, size_t n, Ident *out)
{
    BitReader rdr(d, n);
    uint8_t type;
    int rc = read_header_begin(rdr, &type);
    if (rc) return rc;
    if (type != 1) return LWF_ERR_HEADER_BAD_TYPE;
    uint32_t ver, ch, rate, bmax, bnom, bmin, b0, b1, framing;
    RD(rdr.u(32, &ver));
    if (ver != 0) return LWF_ERR_UNSUPPORTED_VERSION;
    RD(rdr.u(8, &ch));
    RD(rdr.u(32, &rate));
    RD(rdr.u(32, &bmax));
    RD(rdr.u(32, &bnom));
    RD(rdr.u(32, &bmin));
    RD(rdr.u(4, &b0));
    RD(rdr.u(4, &b1));
    RD(rdr.u(8, &framing));
    if (b0 < 6 || b0 > 13 || b1 < 6 || b1 > 13 || framing != 1 || b0 > b1 || ch == 0 || rate == 0) BAD();
    out->audio_channels = (uint8_t)ch;
    out->audio_sample_rate = rate;
    out->bitrate_maximum = (int32_t)bmax;
    out->bitrate_nominal = (int32_t)bnom;
    out->bitrate_minimum = (int32_t)bmin;
    out->blocksize_0 = (uint8_t)b0;
    out->blocksize_1 = (uint8_t)b1;
    return LWB_OK;
}

static bool valid_utf8(const uint8_t *s, size_t n)
{
    size_t i = 0;
    while (i < n) {
        const uint8_t c = s[i];
        size_t extra;
        uint32_t cp;
        if (c < 0x80) { i++; continue; }
        else if ((c & 0xe0) == 0xc0) { extra = 1; cp = c & 0x1f; }
        else if ((c & 0xf0) == 0xe0) { extra = 2; cp = c & 0x0f; }
        else if ((c & 0xf8) == 0xf0) { extra = 3; cp = c & 0x07; }
        else return false;
        if (i + extra >= n) return false;
        for (size_t k = 1; k <= extra; k++) {
            if ((s[i + k] & 0xc0) != 0x80) return false;
            cp = (cp << 6) | (s[i + k] & 0x3f);
        }
        if ((extra == 1 && cp < 0x80) || (extra == 2 && cp < 0x800) || (extra == 3 && cp < 0x10000) || cp > 0x10ffff ||
            (cp >= 0xd800 && cp <= 0xdfff))
            return false;
        i += extra + 1;
    }
    return true;
}

// read_header_comment, header.rs:309-358 (byte-oriented Cursor, little endian)
static int read_comment(const uint8_t *d, size_t n, Headers *h)
{
    BitReader rdr(d, n);
    uint8_t type;
    int rc = read_header_begin(rdr, &type);
    if (rc) return rc;
    if (type != 3) return LWF_ERR_HEADER_BAD_TYPE;
    size_t at = 7;
    auto u32le = [&](uint32_t *v) {
        if (at + 4 > n) return false;
        *v = (uint32_t)d[at] | ((uint32_t)d[at + 1] << 8) | ((uint32_t)d[at + 2] << 16) | ((uint32_t)d[at + 3] << 24);
        at += 4;
        return true;
    };
    uint32_t vlen;
    RD(u32le(&vlen));
    if (at + vlen > n) return LWF_ERR_END_OF_PACKET;
    if (!valid_utf8(d + at, vlen)) return LWF_ERR_UTF8;
    h->vendor.assign((const char *)d + at, vlen);
    at += vlen;
    uint32_t count;
    RD(u32le(&count));
    for (uint32_t i = 0; i < count; i++) {
        uint32_t clen;
        RD(u32le(&clen));
        if (at + clen > n) return LWF_ERR_END_OF_PACKET;
        const uint8_t *c = d + at;
        at += clen;
        if (!valid_utf8(c, clen)) continue;                 // tolerated, header.rs:329-339
        const void *eq = std::memchr(c, '=', clen);
        if (!eq) continue;                                  // tolerated, header.rs:340-345
        const size_t k = (const uint8_t *)eq - c;
        h->comments.emplace_back(std::string((const char *)c, k), std::string((const char *)c + k + 1, clen - k - 1));
    }
    if (at + 1 > n) return LWF_ERR_END_OF_PACKET;
    if (d[at] != 1) BAD();
    return LWB_OK;
}

// header.rs:563-583, 585-608, 616-649
static const uint32_t kMaxBases[32] = {0xffffffff, 0xffffffff, 0x0000ffff, 0x00000659, 0x000000ff, 0x00000054, 0x00000028,
                                       0x00000017, 0x0000000f, 0x0000000b, 0x00000009, 0x00000007, 0x00000006, 0x00000005,
                                       0x00000004, 0x00000004, 3, 3, 3, 3, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2};
static const uint8_t kMaxBaseBits[32] = {0x1f, 0x1f, 0x0f, 0x0a, 0x07, 0x06, 0x05, 0x04, 0x03, 0x03, 0x03, 0x02, 0x02, 0x02, 0x02, 0x02,
                                         1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1};

static uint32_t exp_fast(uint32_t base, uint8_t exponent)
{
    uint32_t res = 1, selfmul = base;
    for (int i = 0; i < 8; i++) {
        if ((1u << i) & exponent) res *= selfmul;
        const uint64_t sq = (uint64_t)selfmul * selfmul;
        if (sq > 0xffffffffull) return res;                 // the reference panics only if the square were needed
        selfmul = (uint32_t)sq;
    }
    return res;
}

static uint32_t lookup1_values(uint32_t entries, uint16_t dimensions)
{
    if (dimensions >= 32) return entries == 0 ? 0 : 1;
    const uint8_t max_bits = kMaxBaseBits[dimensions];
    const uint32_t max_base = kMaxBases[dimensions];
    uint32_t base_bits = 0;
    for (int i = 0; i <= max_bits; i++) {
        const uint32_t bit = 1u << (max_bits - i);
        base_bits |= bit;
        if (max_base < base_bits || exp_fast(base_bits, (uint8_t)dimensions) > entries) base_bits &= ~bit;
    }
    return base_bits;
}

// read_codebook, header.rs:673-768; lookup_vec_val_decode, :495-534
static int read_codebook(BitReader &rdr, Codebook *cb)
{
    uint32_t sync, dims, entries;
    RD(rdr.u(24, &sync));
    if (sync != 0x564342) BAD();
    RD(rdr.u(16, &dims));
    RD(rdr.u(24, &entries));
    bool ordered;
    RD(rdr.flag(&ordered));
    if (entries > LWF_MAX_ENTRIES) return LWB_ERR_BUFFER;
    std::vector<uint8_t> lengths;
    lengths.reserve(entries);
    if (!ordered) {
        bool sparse;
        RD(rdr.flag(&sparse));
        for (uint32_t i = 0; i < entries; i++) {
            uint32_t len = 0;
            if (sparse) {
                bool f;
                RD(rdr.flag(&f));
                if (f) { RD(rdr.u(5, &len)); len += 1; }
            } else {
                RD(rdr.u(5, &len));
                len += 1;
            }
            lengths.push_back((uint8_t)len);
        }
    } else {
        uint32_t cur = 0, len;
        RD(rdr.u(5, &len));
        len += 1;
        while (cur < entries) {
            uint32_t number;
            RD(rdr.u(ilog(entries - cur), &number));
            for (uint32_t k = 0; k < number; k++) lengths.push_back((uint8_t)len);
            cur += number;
            len += 1;
            if (cur > entries) BAD();
        }
    }
    uint32_t lookup_type;
    RD(rdr.u(4, &lookup_type));
    if (lookup_type > 2) BAD();
    cb->dimensions = (uint16_t)dims;
    if (lookup_type != 0) {
        uint32_t raw_min, raw_delta, vbits;
        RD(rdr.u(32, &raw_min));
        RD(rdr.u(32, &raw_delta));
        const float minimum = float32_unpack(raw_min), delta = float32_unpack(raw_delta);
        RD(rdr.u(4, &vbits));
        vbits += 1;
        bool sequence_p;
        RD(rdr.flag(&sequence_p));
        const uint64_t lookup_values = lookup_type == 1 ? lookup1_values(entries, (uint16_t)dims) : (uint64_t)entries * dims;
        // convert_to_usize! / BufferNotAddressable (header.rs:117-125): refuse tables no host can hold
        if (lookup_values > LWF_MAX_VQ_ELEMS || (uint64_t)entries * dims > LWF_MAX_VQ_ELEMS) return LWB_ERR_BUFFER;
        std::vector<uint32_t> mult;
        mult.reserve((size_t)lookup_values);
        for (uint64_t i = 0; i < lookup_values; i++) {
            uint32_t m;
            RD(rdr.u(vbits, &m));
            mult.push_back(m);
        }
        cb->has_vq = true;
        cb->vq.reserve((size_t)entries * dims);
        if (lookup_type == 1) {
            const size_t lv = mult.size();
            for (uint32_t off = 0; off < entries; off++) {
                float last = 0.f;
                size_t divisor = 1;
                for (uint32_t k = 0; k < dims; k++) {
                    // with lv == 0 the reference divides by zero (panic); such a book has no entries to decode
                    const size_t mo = lv ? (size_t)(off / (uint32_t)divisor) % lv : 0;
                    const float e = (float)(lv ? mult[mo] : 0) * delta + minimum + last;
                    if (sequence_p) last = e;
                    cb->vq.push_back(e);
                    divisor *= lv;
                }
            }
        } else {
            for (uint32_t off = 0; off < entries; off++) {
                float last = 0.f;
                size_t mo = (size_t)off * dims;
                for (uint32_t k = 0; k < dims; k++) {
                    const float e = (float)mult[mo] * delta + minimum + last;
                    if (sequence_p) last = e;
                    cb->vq.push_back(e);
                    mo++;
                }
            }
        }
    }
    if (cb->tree.load(lengths) != HUFF_OK) BAD();          // From<HuffmanError>, header.rs:74-78
    return LWB_OK;
}

// header_cached.rs:129-158
static inline float bark(float x)
{
    return 13.1f * atanf(0.00074f * x) + 2.24f * atanf(0.0000000185f * x * x) + 0.0001f * x;
}
// (also generates the tables lwb_setup_set_floor0 is not given, lwb_api.cu)
std::vector<float> bark_map_cos_omega(uint16_t n, uint16_t rate, uint16_t bark_map_size)
{
    std::vector<float> res;
    res.reserve(n);
    const float hfl = (float)rate / 2.0f;
    const float hfl_dn = hfl / (float)n;
    const float const_part = (float)bark_map_size / bark(hfl);
    const float bms_m1 = (float)bark_map_size - 1.0f;
    const float omega_factor = 3.14159265358979323846f / (float)bark_map_size;
    for (uint32_t i = 0; i < n; i++) {
        const float fb = floorf(bark((float)i * hfl_dn) * const_part);
        const float map_elem = fminf(fb, bms_m1);
        res.push_back(cosf(map_elem * omega_factor));
    }
    return res;
}

// read_floor, header.rs:771-920
static int read_floor(BitReader &rdr, uint16_t codebook_cnt, uint8_t bs0, uint8_t bs1, Floor *fl)
{
    uint32_t type;
    RD(rdr.u(16, &type));
    if (type == 0) {
        uint32_t order, rate, bms, abits, aoff, nbooks;
        RD(rdr.u(8, &order));
        RD(rdr.u(16, &rate));
        RD(rdr.u(16, &bms));
        RD(rdr.u(6, &abits));
        if (abits > 64) BAD();
        RD(rdr.u(8, &aoff));
        RD(rdr.u(4, &nbooks));
        nbooks += 1;
        fl->type = 0;
        Floor0 &f = fl->f0;
        f.order = (uint8_t)order;
        f.amplitude_bits = (uint8_t)abits;
        f.amplitude_offset = (uint8_t)aoff;
        f.number_of_books = (uint8_t)nbooks;
        f.rate = (uint16_t)rate;
        f.bark_map_size = (uint16_t)bms;
        for (uint32_t i = 0; i < nbooks; i++) {
            uint32_t v;
            RD(rdr.u(8, &v));
            if (v > codebook_cnt) BAD();                    // `>`: the reference's check, header.rs:796
            f.book_list.push_back((uint8_t)v);
        }
        f.bark_cos_omega[0] = bark_map_cos_omega((uint16_t)(1u << (bs0 - 1)), (uint16_t)rate, (uint16_t)bms);
        f.bark_cos_omega[1] = bark_map_cos_omega((uint16_t)(1u << (bs1 - 1)), (uint16_t)rate, (uint16_t)bms);
        return LWB_OK;
    }
    if (type != 1) BAD();
    fl->type = 1;
    Floor1 &f = fl->f1;
    uint32_t partitions;
    RD(rdr.u(5, &partitions));
    int max_class = -1;
    for (uint32_t i = 0; i < partitions; i++) {
        uint32_t c;
        RD(rdr.u(4, &c));
        max_class = std::max(max_class, (int)c);
        f.partition_class.push_back((uint8_t)c);
    }
    for (int c = 0; c <= max_class; c++) {
        uint32_t dim, sub;
        RD(rdr.u(3, &dim));
        f.class_dimensions.push_back((uint8_t)(dim + 1));
        RD(rdr.u(2, &sub));
        f.class_subclasses.push_back((uint8_t)sub);
        if (sub != 0) {
            uint32_t mb;
            RD(rdr.u(8, &mb));
            if (mb >= codebook_cnt) BAD();
            f.class_masterbooks.push_back((uint8_t)mb);
        } else {
            f.class_masterbooks.push_back(0);
        }
        std::vector<int16_t> books;
        for (uint32_t k = 0; k < (1u << sub); k++) {
            uint32_t b;
            RD(rdr.u(8, &b));
            const int16_t book = (int16_t)b - 1;
            if (book >= (int16_t)codebook_cnt) BAD();
            books.push_back(book);
        }
        f.subclass_books.push_back(std::move(books));
    }
    uint32_t mult, rangebits;
    RD(rdr.u(2, &mult));
    f.multiplier = (uint8_t)(mult + 1);
    RD(rdr.u(4, &rangebits));
    uint32_t values = 2;
    for (uint8_t c : f.partition_class) values += f.class_dimensions[c];
    if (values > 65) BAD();
    f.x_list.push_back(0);
    f.x_list.push_back(1u << rangebits);
    for (uint8_t c : f.partition_class)
        for (uint8_t k = 0; k < f.class_dimensions[c]; k++) {
            uint32_t x;
            RD(rdr.u(rangebits, &x));
            f.x_list.push_back(x);
        }
    // uniqueness (header.rs:887-901): sorted, no two equal; the scan starts with last = 1, so an
    // x value of 1 directly after the leading 0 ... is compared against the previous element only
    std::vector<uint32_t> sorted(f.x_list);
    std::stable_sort(sorted.begin(), sorted.end());
    uint32_t last = 1;
    for (uint32_t x : sorted) {
        if (x == last) BAD();
        last = x;
    }
    return LWB_OK;
}

// read_residue, header.rs:922-983; ResidueBook::read_book, :445-468 (reads 7 of the 8 cascade bits)
static int read_residue(BitReader &rdr, const std::vector<Codebook> &codebooks, Residue *r)
{
    uint32_t type, begin, end, psize, classes, classbook;
    RD(rdr.u(16, &type));
    if (type > 2) BAD();
    RD(rdr.u(24, &begin));
    RD(rdr.u(24, &end));
    if (begin > end) BAD();
    RD(rdr.u(24, &psize));
    RD(rdr.u(6, &classes));
    RD(rdr.u(8, &classbook));
    classes += 1;
    std::vector<uint8_t> cascade;
    for (uint32_t i = 0; i < classes; i++) {
        uint32_t low, high = 0;
        bool f;
        RD(rdr.u(3, &low));
        RD(rdr.flag(&f));
        if (f) RD(rdr.u(5, &high));
        cascade.push_back((uint8_t)((high << 3) | low));
    }
    for (uint8_t c : cascade) {
        ResidueBook b;
        b.vals_used = c;
        for (int i = 0; i < 7; i++) {
            if (!(c & (1 << i))) continue;
            uint32_t v;
            RD(rdr.u(8, &v));
            if (v >= codebooks.size() || !codebooks[v].has_vq) BAD();
            b.val[i] = (uint8_t)v;
        }
        r->books.push_back(b);
    }
    if (classbook >= codebooks.size()) BAD();
    r->type = (uint8_t)type;
    r->begin = begin;
    r->end = end;
    r->partition_size = psize + 1;
    r->classifications = (uint8_t)classes;
    r->classbook = (uint8_t)classbook;
    return LWB_OK;
}

// read_mapping, header.rs:985-1058
static int read_mapping(BitReader &rdr, uint8_t chan_ilog, uint8_t channels, uint8_t floor_count, uint8_t residue_count, Mapping *m)
{
    uint32_t type;
    RD(rdr.u(16, &type));
    if (type > 0) BAD();
    bool f;
    uint32_t submaps = 1, steps = 0;
    RD(rdr.flag(&f));
    if (f) { RD(rdr.u(4, &submaps)); submaps += 1; }
    RD(rdr.flag(&f));
    if (f) { RD(rdr.u(8, &steps)); steps += 1; }
    for (uint32_t i = 0; i < steps; i++) {
        uint32_t mag, ang;
        RD(rdr.u(chan_ilog, &mag));
        RD(rdr.u(chan_ilog, &ang));
        if (ang == mag || mag >= channels || ang >= channels) BAD();
        m->magnitudes.push_back((uint8_t)mag);
        m->angles.push_back((uint8_t)ang);
    }
    uint32_t reserved;
    RD(rdr.u(2, &reserved));
    if (reserved != 0) BAD();
    if (submaps > 1) {
        for (uint32_t c = 0; c < channels; c++) {
            uint32_t v;
            RD(rdr.u(4, &v));
            if (v >= submaps) BAD();
            m->mux.push_back((uint8_t)v);
        }
    } else {
        m->mux.assign(channels, 0);
    }
    for (uint32_t s = 0; s < submaps; s++) {
        uint32_t skip, fl, rs;
        RD(rdr.u(8, &skip));
        RD(rdr.u(8, &fl));
        RD(rdr.u(8, &rs));
        if (fl >= floor_count || rs >= residue_count) BAD();
        m->submap_floors.push_back((uint8_t)fl);
        m->submap_residues.push_back((uint8_t)rs);
    }
    return LWB_OK;
}

// read_header_setup, header.rs:1082-1155; read_mode_info, :1060-1077
static int read_setup(const uint8_t *d, size_t n, Headers *h)
{
    BitReader rdr(d, n);
    uint8_t type;
    int rc = read_header_begin(rdr, &type);
    if (rc) return rc;
    if (type != 5) return LWF_ERR_HEADER_BAD_TYPE;
    const uint8_t channels = h->ident.audio_channels;
    const uint8_t chan_ilog = ilog((uint64_t)(channels - 1));
    uint32_t v;
    RD(rdr.u(8, &v));
    const uint16_t codebook_cnt = (uint16_t)(v + 1);
    h->codebooks.resize(codebook_cnt);
    for (auto &cb : h->codebooks)
        if ((rc = read_codebook(rdr, &cb))) return rc;
    RD(rdr.u(6, &v));
    for (uint32_t i = 0; i < v + 1; i++) {
        uint32_t t;
        RD(rdr.u(16, &t));
        if (t != 0) BAD();
    }
    RD(rdr.u(6, &v));
    const uint8_t floor_count = (uint8_t)(v + 1);
    h->floors.resize(floor_count);
    for (auto &fl : h->floors)
        if ((rc = read_floor(rdr, codebook_cnt, h->ident.blocksize_0, h->ident.blocksize_1, &fl))) return rc;
    RD(rdr.u(6, &v));
    const uint8_t residue_count = (uint8_t)(v + 1);
    h->residues.resize(residue_count);
    for (auto &r : h->residues)
        if ((rc = read_residue(rdr, h->codebooks, &r))) return rc;
    RD(rdr.u(6, &v));
    const uint8_t mapping_count = (uint8_t)(v + 1);
    h->mappings.resize(mapping_count);
    for (auto &m : h->mappings)
        if ((rc = read_mapping(rdr, chan_ilog, channels, floor_count, residue_count, &m))) return rc;
    RD(rdr.u(6, &v));
    const uint8_t mode_count = (uint8_t)(v + 1);
    for (uint32_t i = 0; i < mode_count; i++) {
        bool bf;
        uint32_t wt, tt, mp;
        RD(rdr.flag(&bf));
        RD(rdr.u(16, &wt));
        RD(rdr.u(16, &tt));
        RD(rdr.u(8, &mp));
        if (wt != 0 || tt != 0 || mp >= mapping_count) BAD();
        ModeInfo mi;
        mi.blockflag = bf;
        mi.mapping = (uint8_t)mp;
        h->modes.push_back(mi);
    }
    bool framing;
    RD(rdr.flag(&framing));
    if (!framing) BAD();
    return LWB_OK;
}

// ---------------------------------------------------------------------------------------------
// audio.rs front half
// ---------------------------------------------------------------------------------------------
enum { FL_OK = 0, FL_UNUSED = 1, FL_UNDECODABLE = 2 };

// read_huffman_vq, header.rs:546-560: 0 ok, 1 end of packet, 2 no value mapping
static int read_huffman_vq(BitReader &rdr, const Codebook &cb, const float **vec)
{
    uint32_t idx;
    if (!cb.tree.read(rdr, &idx)) return 1;
    if (!cb.has_vq) return 2;
    *vec = cb.vq.data() + (size_t)idx * cb.dimensions;
    return 0;
}

// floor_zero_decode, audio.rs:109-158: cosines of the coefficients + amplitude
static int floor0_decode(BitReader &rdr, const std::vector<Codebook> &codebooks, const Floor0 &fl, std::vector<float> *coeff,
                         uint64_t *amplitude)
{
    if (!rdr.read(fl.amplitude_bits, amplitude)) return FL_UNUSED;
    if (*amplitude == 0) return FL_UNUSED;
    uint32_t booknumber;
    if (!rdr.u(ilog(fl.number_of_books), &booknumber)) return FL_UNUSED;
    if (booknumber >= fl.book_list.size()) return FL_UNDECODABLE;
    const size_t bi = fl.book_list[booknumber];
    if (bi >= codebooks.size()) return FL_UNDECODABLE;      // the reference indexes out of bounds here (header check is `>`)
    const Codebook &cb = codebooks[bi];
    // floor0_order < 2: the reference's curve computation underflows `(order - 3) / 2` / `(order - 2) / 2` and
    // panics on the slice index (audio.rs:178-186); a hostile header must not get further than this
    if (fl.order < 2) return FL_UNDECODABLE;
    coeff->clear();
    float last = 0.f;
    for (;;) {
        float last_new = last;
        const float *tv;
        const int rc = read_huffman_vq(rdr, cb, &tv);
        if (rc == 1) return FL_UNUSED;
        if (rc == 2) return FL_UNDECODABLE;
        for (uint32_t k = 0; k < cb.dimensions; k++) {
            coeff->push_back(cosf(last + tv[k]));
            last_new = tv[k];
            if (coeff->size() == fl.order) return FL_OK;
        }
        last += last_new;
        if (coeff->size() >= fl.order) return FL_OK;
        if (cb.dimensions == 0) return FL_UNDECODABLE;      // would loop forever in the reference
    }
}

// floor_zero_compute_curve, audio.rs:160-212
static void floor0_curve(const std::vector<float> &cosc, uint64_t amplitude, const Floor0 &fl, bool blockflag, uint32_t n, float *out)
{
    const std::vector<float> &bark_cos = fl.bark_cos_omega[blockflag ? 1 : 0];
    const uint64_t max_amp = fl.amplitude_bits >= 64 ? ~0ull : (((uint64_t)1 << fl.amplitude_bits) - 1);   // 64 bits are legal (header.rs:780-787)
    const float common = (float)amplitude * (float)fl.amplitude_offset / (float)max_amp;
    size_t i = 0;
    size_t w = 0;
    while (i < n) {
        const float cos_omega = bark_cos[i];
        size_t pu, qu;
        float p, q;
        if (fl.order & 1) {
            pu = ((size_t)fl.order - 3) / 2;
            qu = ((size_t)fl.order - 1) / 2;
            p = 1.0f - cos_omega * cos_omega;
            q = 0.25f;
        } else {
            pu = qu = ((size_t)fl.order - 2) / 2;
            p = (1.0f - cos_omega) / 2.0f;
            q = (1.0f + cos_omega) / 2.0f;
        }
        for (size_t j = 0; j <= pu; j++) {
            const float pm = cosc[2 * j + 1] - cos_omega;
            p *= 4.0f * pm * pm;
        }
        for (size_t j = 0; j <= qu; j++) {
            const float qm = cosc[2 * j] - cos_omega;
            q *= 4.0f * qm * qm;
        }
        const float lfv = expf(0.11512925f * (common / sqrtf(p + q) - (float)fl.amplitude_offset));
        float cond = cos_omega;
        while (cos_omega == cond) {
            out[w++] = lfv;
            i++;
            if (i >= bark_cos.size()) break;
            cond = bark_cos[i];
        }
        if (i >= bark_cos.size()) break;
    }
    for (; w < n; w++) out[w] = 0.f;
}

// Whether a type-0 floor can travel as an LWB_FLOOR_ZERO record (lwf_packet_decode_ex with LWF_DECODE_FLOOR0_RECORDS):
// the record holds at most LWB_MAX_POSTS - 2 coefficients, and lwb_setup_set_floor0 takes the floor (a zero rate or
// bark map size gives a NaN bark table, on which the reference's run walk never ends).
static bool floor0_record_ok(const Floor0 &fl)
{
    return fl.order >= 2 && fl.order <= LWB_MAX_POSTS - 2 && fl.rate && fl.bark_map_size;
}

// floor_one_decode, audio.rs:215-251
static int floor1_decode(BitReader &rdr, const std::vector<Codebook> &codebooks, const Floor1 &fl, uint32_t *y, uint32_t *count)
{
    bool nonzero;
    if (!rdr.flag(&nonzero)) return FL_UNUSED;
    if (!nonzero) return FL_UNUSED;
    static const uint32_t ranges[4] = {256, 128, 86, 64};
    const uint8_t b = ilog(ranges[fl.multiplier - 1] - 1);
    uint32_t n = 0, v;
    if (!rdr.u(b, &v)) return FL_UNUSED;
    y[n++] = v;
    if (!rdr.u(b, &v)) return FL_UNUSED;
    y[n++] = v;
    for (uint8_t cls : fl.partition_class) {
        const uint8_t cdim = fl.class_dimensions[cls], cbits = fl.class_subclasses[cls];
        const uint32_t csub = (1u << cbits) - 1;
        uint32_t cval = 0;
        if (cbits > 0)
            if (!codebooks[fl.class_masterbooks[cls]].tree.read(rdr, &cval)) return FL_UNUSED;
        for (uint8_t k = 0; k < cdim; k++) {
            const int16_t book = fl.subclass_books[cls][cval & csub];
            cval >>= cbits;
            if (book >= 0) {
                if (!codebooks[(size_t)book].tree.read(rdr, &v)) return FL_UNUSED;
                y[n++] = v;
            } else {
                y[n++] = 0;
            }
        }
    }
    *count = n;
    return FL_OK;
}

// LWB_ENTRY_VQ: instead of adding the VQ vectors into dense residue vectors on the host, the decode emits, per
// residue_packet_read_partition call, one RUN ("codebook b, pass p, starting at position x") and one 16-bit entry per
// vector; the device does the additions in the same order.
struct VqSink {
    lwb_vq_run *runs = nullptr;
    uint16_t *entries = nullptr;
    size_t run_cap = 0, ent_cap = 0, n_runs = 0, n_ent = 0;
    bool overflow = false;
    // context of the residue decode in progress
    size_t base = 0;                  // position of vec_v[0]: channel * n/2 + offset (types 0 / 1) or the interleaved index (type 2)
    uint8_t pass = 0, kind = 0, aux = 0, book = 0;
    int cur = -1;                     // run being filled
    void begin() { cur = -1; }
    // vector number `i` of the partition (its position = base + i * (kind == 1 ? 1 : dims)) holds `entry`
    void put(uint32_t entry, size_t i, size_t dims)
    {
        const size_t pos = base + i * (kind == 1 ? 1 : dims);
        if (entry > 0xffffu || pos > 0xffffu || n_ent >= ent_cap || n_ent > 0xffffu) { overflow = true; return; }
        if (cur < 0 || runs[cur].count == 255) {
            if (n_runs >= run_cap) { overflow = true; return; }
            cur = (int)n_runs++;
            lwb_vq_run &r = runs[cur];
            r.pos = (uint16_t)pos;
            r.first = (uint16_t)n_ent;
            r.book = book;
            r.pass_kind = LWB_VQ_PASS_KIND(pass, kind);
            r.aux = aux;
            r.count = 0;
        }
        runs[cur].count++;
        entries[n_ent++] = (uint16_t)entry;
    }
};

// residue_packet_read_partition, audio.rs:588-619 with the additions left to the device: 0 ok, 1 end of packet
static int residue_partition_vq(BitReader &rdr, const Codebook &cb, const Residue &r, size_t vlen, VqSink &sink)
{
    // The loop bounds and early exits are residue_partition's; per symbol only the codeword is read and its entry stored
    // (positions advance by a constant, the run header is written once per 255 entries).
    uint32_t idx;
    sink.begin();
    const size_t dims = cb.dimensions;
    if (r.type == 0) {
        if (dims == 0) return 0;
        const size_t step = r.partition_size / dims;
        const bool fits = (dims - 1) * step < vlen;          // i + (dims - 1) * step >= vlen first fails at i = vlen - (dims - 1) * step
        const size_t ok_until = fits ? vlen - (dims - 1) * step : 0;
        for (size_t i = 0; i < step; i++) {
            if (!cb.tree.read(rdr, &idx)) return 1;
            if (i >= ok_until) return 0;                     // (slice index out of range: a panic in the reference)
            sink.put(idx, i, dims);
        }
    } else {
        const size_t psize = r.partition_size;
        size_t i = 0, v = 0;
        while (i < psize) {
            if (!cb.tree.read(rdr, &idx)) return 1;
            if (i + dims > vlen) break;
            if (dims == 0) break;
            sink.put(idx, v, dims);
            i += dims;
            v++;
        }
    }
    return 0;
}

// residue_packet_read_partition, audio.rs:588-619: 0 ok, 1 end of packet
static int residue_partition(BitReader &rdr, const Codebook &cb, const Residue &r, float *v, size_t vlen)
{
    const float *e;
    if (r.type == 0) {
        const size_t dims = cb.dimensions;
        if (dims == 0) return 0;                            // division by zero in the reference
        const size_t step = r.partition_size / dims;
        for (size_t i = 0; i < step; i++) {
            const int rc = read_huffman_vq(rdr, cb, &e);
            if (rc) return 1;
            for (size_t j = 0; j < dims; j++) {
                if (i + j * step >= vlen) return 0;         // slice index out of range panics in the reference
                v[i + j * step] += e[j];
            }
        }
    } else {
        const size_t psize = r.partition_size;
        size_t i = 0;
        while (i < psize) {
            const int rc = read_huffman_vq(rdr, cb, &e);
            if (rc) return 1;
            if (i + cb.dimensions > vlen) break;
            for (size_t k = 0; k < cb.dimensions; k++) v[i + k] += e[k];
            i += cb.dimensions;
            if (cb.dimensions == 0) break;
        }
    }
    return 0;
}

// residue_packet_decode_inner, audio.rs:621-716.  `vectors`: [ch][blocksize/2], zeroed here.
// sink != nullptr: VQ records instead of additions (chbase[j] = position of channel j's vector; kind / aux set by the caller)
static int residue_decode_inner(BitReader &rdr, uint32_t cur_blocksize, const std::vector<uint8_t> &dnd, const Residue &r,
                                const std::vector<Codebook> &codebooks, std::vector<float> &vectors, VqSink *sink = nullptr,
                                const size_t *chbase = nullptr)
{
    const size_t ch = dnd.size(), actual = cur_blocksize / 2;
    const size_t lim_begin = std::min<size_t>(r.begin, actual), lim_end = std::min<size_t>(r.end, actual);
    const Codebook &classbook = codebooks[r.classbook];
    const size_t cpc = classbook.dimensions;
    const size_t n_to_read = lim_end - lim_begin;
    const size_t parts = n_to_read / r.partition_size;
    if (!sink) vectors.assign(ch * actual, 0.f);
    if (n_to_read == 0) return 0;
    if (cpc == 0) return 1;
    const size_t stride = parts + cpc;
    thread_local std::vector<uint32_t> cls;                 // scratch reused across packets (no allocation per packet)
    cls.assign(ch * stride, 0);
    unsigned passes_used = 1;                               // pass 0 reads the classifications
    for (const ResidueBook &rb : r.books) passes_used |= rb.vals_used;
    for (int pass = 0; pass < 8; pass++) {
        if (!(passes_used & (1u << pass))) continue;         // no class has a book in this pass: nothing is read
        size_t pc = 0;
        while (pc < parts) {
            if (pass == 0) {
                for (size_t j = 0; j < ch; j++) {
                    if (dnd[j]) continue;
                    uint32_t temp;
                    if (!classbook.tree.read(rdr, &temp)) return 0;           // end of packet is normal
                    for (size_t i = cpc; i-- > 0;) {
                        cls[j * stride + i + pc] = temp % r.classifications;
                        temp /= r.classifications;
                    }
                }
            }
            for (size_t k = 0; k < cpc; k++) {
                if (pc >= parts) break;
                for (size_t j = 0; j < ch; j++) {
                    if (dnd[j]) continue;
                    const size_t offs = lim_begin + pc * r.partition_size;
                    const uint32_t vqclass = cls[j * stride + pc];
                    const ResidueBook &rb = r.books[vqclass];
                    if (rb.vals_used & (1u << pass)) {
                        const Codebook &cb = codebooks[rb.val[pass]];
                        if (!cb.has_vq) return 1;           // the reference panics ("must have a value mapping")
                        if (sink) {
                            sink->pass = (uint8_t)pass;
                            sink->book = rb.val[pass];
                            sink->base = chbase[j] + offs;
                            if (residue_partition_vq(rdr, cb, r, actual - offs, *sink)) return 0;
                        } else if (residue_partition(rdr, cb, r, vectors.data() + j * actual + offs, actual - offs)) return 0;
                    }
                }
                pc++;
            }
        }
    }
    return 0;
}

// residue_packet_decode, audio.rs:721-760
// sink != nullptr: records; chbase[j] = position of submap channel j's vector, residue_idx / submap go into the records
static int residue_decode(BitReader &rdr, uint32_t cur_blocksize, const std::vector<uint8_t> &dnd, const Residue &r,
                          const std::vector<Codebook> &codebooks, std::vector<float> &out, VqSink *sink = nullptr,
                          const size_t *chbase = nullptr, uint8_t residue_idx = 0, uint8_t submap = 0)
{
    const size_t ch = dnd.size(), vec = cur_blocksize / 2;
    if (r.type != 2) {
        if (sink) { sink->kind = r.type == 0 ? 1 : 0; sink->aux = residue_idx; }
        return residue_decode_inner(rdr, cur_blocksize, dnd, r, codebooks, out, sink, chbase);
    }
    bool any = false;
    for (uint8_t d : dnd) any |= !d;
    if (!any) {
        if (!sink) out.assign(ch * vec, 0.f);
        return 0;
    }
    if (sink) {                      // one interleaved vector for the whole submap; the device de-interleaves
        thread_local std::vector<uint8_t> one1(1, 0);
        const size_t zero = 0;
        sink->kind = 2;
        sink->aux = submap;
        const uint32_t bs2s = (uint32_t)(uint16_t)(cur_blocksize * ch);
        return residue_decode_inner(rdr, bs2s, one1, r, codebooks, out, sink, &zero);
    }
    thread_local std::vector<uint8_t> one(1, 0);
    thread_local std::vector<float> inter;
    // cur_blocksize * ch as u16: the product wraps at 16 bits in the reference
    const uint32_t bs2 = (uint32_t)(uint16_t)(cur_blocksize * ch);
    if (residue_decode_inner(rdr, bs2, one, r, codebooks, inter)) return 1;
    out.assign(ch * vec, 0.f);
    for (size_t j = 0; j < ch; j++)
        for (size_t i = 0; i < vec; i++) {
            const size_t src = i * ch + j;
            if (src < inter.size()) out[j * vec + i] = inter[src];
        }
    return 0;
}

struct PacketHead { uint8_t mode; bool blockflag; bool prev, next; uint32_t n; };

// audio.rs:921-939 (and :877-888)
static int packet_head(const Headers &h, BitReader &rdr, PacketHead *ph)
{
    bool is_header;
    if (!rdr.flag(&is_header)) return LWF_ERR_END_OF_PACKET;
    if (is_header) return LWF_ERR_AUDIO_IS_HEADER;
    uint32_t mode;
    if (!rdr.u(ilog((uint64_t)h.modes.size() - 1), &mode)) return LWF_ERR_END_OF_PACKET;
    if (mode >= h.modes.size()) return LWB_ERR_BAD_FORMAT;
    ph->mode = (uint8_t)mode;
    ph->blockflag = h.modes[mode].blockflag;
    ph->n = 1u << (ph->blockflag ? h.ident.blocksize_1 : h.ident.blocksize_0);
    ph->prev = ph->next = true;
    if (ph->blockflag) {
        if (!rdr.flag(&ph->prev)) return LWF_ERR_END_OF_PACKET;
        if (!rdr.flag(&ph->next)) return LWF_ERR_END_OF_PACKET;
    }
    return LWB_OK;
}

// records: type-0 floors that qualify (floor0_record_ok) come out as LWB_FLOOR_ZERO records in their floor1_y row instead
// of dense curves.
static int packet_decode(const Headers &h, const uint8_t *packet, size_t len, lwf_decoded_packet *out, VqSink *sink = nullptr,
                         bool records = false)
{
    BitReader rdr(packet, len);
    PacketHead ph;
    int rc = packet_head(h, rdr, &ph);
    if (rc) return rc;
    const ModeInfo &mode = h.modes[ph.mode];
    const Mapping &mp = h.mappings[mode.mapping];
    const size_t C = h.ident.audio_channels, n2 = ph.n / 2;
    out->mode_number = ph.mode;
    out->blockflag = ph.blockflag;
    out->prev_window_flag = ph.prev;
    out->next_window_flag = ph.next;
    out->n = ph.n;
    // floor_decode, audio.rs:557-586
    thread_local std::vector<uint8_t> no_residue;
    thread_local std::vector<float> cosc;
    no_residue.assign(C, 0);
    for (size_t c = 0; c < C; c++) {
        const Floor &fl = h.floors[mp.submap_floors[mp.mux[c]]];
        int fr;
        if (fl.type == 0) {
            uint64_t amp = 0;
            fr = floor0_decode(rdr, h.codebooks, fl.f0, &cosc, &amp);
            if (fr == FL_OK && records && floor0_record_ok(fl.f0)) {
                // the record: amplitude (low word first), then the coefficient cosines' bits (lewton_b200.h LWB_FLOOR_ZERO)
                uint32_t *y = out->floor1_y + c * LWB_MAX_POSTS;
                std::memset(y, 0, sizeof(uint32_t) * LWB_MAX_POSTS);
                y[0] = (uint32_t)amp;
                y[1] = (uint32_t)(amp >> 32);
                std::memcpy(y + 2, cosc.data(), cosc.size() * sizeof(float));
                out->floor_kind[c] = LWB_FLOOR_ZERO;
            } else if (fr == FL_OK) {
                out->floor_kind[c] = LWB_FLOOR_DENSE;
                floor0_curve(cosc, amp, fl.f0, ph.blockflag, (uint32_t)n2, out->dense_floor + c * n2);
            }
        } else {
            uint32_t cnt = 0;
            uint32_t *y = out->floor1_y + c * LWB_MAX_POSTS;
            std::memset(y, 0, sizeof(uint32_t) * LWB_MAX_POSTS);
            fr = floor1_decode(rdr, h.codebooks, fl.f1, y, &cnt);
            if (fr == FL_OK) out->floor_kind[c] = LWB_FLOOR_ONE;
        }
        if (fr == FL_UNDECODABLE) return LWF_ERR_END_OF_PACKET;  // floor_decode's Err(()) goes through From<()> (audio.rs:46-50)
        if (fr == FL_UNUSED) out->floor_kind[c] = LWB_FLOOR_UNUSED;
        no_residue[c] = fr == FL_UNUSED;
    }
    // audio.rs:944-955
    for (size_t s = 0; s < mp.magnitudes.size(); s++) {
        const uint8_t m = mp.magnitudes[s], a = mp.angles[s];
        if (!(no_residue[m] && no_residue[a])) no_residue[m] = no_residue[a] = 0;
    }
    // audio.rs:957-986
    thread_local std::vector<uint8_t> dnd;
    thread_local std::vector<float> vectors;
    for (size_t i = 0; i < mp.submap_residues.size(); i++) {
        dnd.clear();
        for (size_t j = 0; j < C; j++)
            if (mp.mux[j] == i) dnd.push_back(no_residue[j]);
        const Residue &r = h.residues[mp.submap_residues[i]];
        if (sink) {
            thread_local std::vector<size_t> chbase;
            chbase.clear();
            for (size_t j = 0; j < C; j++)
                if (mp.mux[j] == i) chbase.push_back(j * n2);
            if (residue_decode(rdr, ph.n, dnd, r, h.codebooks, vectors, sink, chbase.data(), mp.submap_residues[i], (uint8_t)i)) return LWB_ERR_BAD_FORMAT;
            continue;
        }
        if (residue_decode(rdr, ph.n, dnd, r, h.codebooks, vectors)) return LWB_ERR_BAD_FORMAT;
        size_t chn = 0;
        for (size_t j = 0; j < C; j++)
            if (mp.mux[j] == i) {
                std::memcpy(out->residue + j * n2, vectors.data() + n2 * chn, n2 * sizeof(float));
                chn++;
            }
    }
    return LWB_OK;
}

// ---------------------------------------------------------------------------------------------
// Ogg paging: what ogg 0.8.0's PacketReader hands to inside_ogg.rs (packets with stream serial,
// page granule position and first/last flags).  RFC 3533 framing, CRC-32 poly 0x04c11db7.
// ---------------------------------------------------------------------------------------------
struct CrcTable {
    uint32_t t[256];
    CrcTable()
    {
        for (uint32_t i = 0; i < 256; i++) {
            uint32_t r = i << 24;
            for (int k = 0; k < 8; k++) r = (r & 0x80000000u) ? (r << 1) ^ 0x04c11db7u : r << 1;
            t[i] = r;
        }
    }
};
static uint32_t ogg_crc(const uint8_t *d, size_t n, size_t crc_at)
{
    static const CrcTable table;              // initialised once, thread-safe (readers on several host threads)
    uint32_t c = 0;
    for (size_t i = 0; i < n; i++) {
        const uint8_t b = (i >= crc_at && i < crc_at + 4) ? 0 : d[i];
        c = (c << 8) ^ table.t[((c >> 24) ^ b) & 0xff];
    }
    return c;
}

struct OggStreamState { std::vector<uint8_t> partial; bool in_packet = false; bool seen = false; bool ended = false;
                        bool drop_continued = false; };   // after a seek: the tail of a packet begun on an earlier page is dropped

struct Ogg {
    const uint8_t *d;
    size_t len, at = 0;
    struct Pending { std::vector<uint8_t> data; uint32_t serial; uint64_t absgp; bool first_stream, last_stream, first_page, last_page; };
    std::vector<Pending> queue;
    size_t qhead = 0;
    std::vector<std::pair<uint32_t, OggStreamState>> streams;
    std::vector<uint8_t> current;

    OggStreamState &state(uint32_t serial)
    {
        for (auto &s : streams)
            if (s.first == serial) return s.second;
        streams.emplace_back(serial, OggStreamState());
        return streams.back().second;
    }

    struct PageHead { uint8_t htype; uint64_t absgp; uint32_t serial, crc; size_t nseg, total; };

    // The header of the page at byte `pos`: LWF_ERR_OGG unless its capture pattern, version, segment table and body are
    // all there
    int page_head(size_t pos, PageHead *h) const
    {
        if (pos + 27 > len) return LWF_ERR_OGG;
        const uint8_t *p = d + pos;
        if (std::memcmp(p, "OggS", 4) != 0 || p[4] != 0) return LWF_ERR_OGG;
        auto le = [p](int at, int n) {
            uint64_t v = 0;
            for (int i = n - 1; i >= 0; i--) v = (v << 8) | p[at + i];
            return v;
        };
        h->htype = p[5];
        h->absgp = le(6, 8);
        h->serial = (uint32_t)le(14, 4);
        h->crc = (uint32_t)le(22, 4);
        h->nseg = p[26];
        if (pos + 27 + h->nseg > len) return LWF_ERR_OGG;
        size_t body = 0;
        for (size_t i = 0; i < h->nseg; i++) body += p[27 + i];
        h->total = 27 + h->nseg + body;
        if (pos + h->total > len) return LWF_ERR_OGG;
        return LWB_OK;
    }

    // parse one page into the queue; LWF_ERR_NO_MORE_PACKETS at the end of the data
    int read_page()
    {
        if (at >= len) return LWF_ERR_NO_MORE_PACKETS;
        PageHead h;
        if (page_head(at, &h)) return LWF_ERR_OGG;
        const uint8_t *p = d + at;
        if (ogg_crc(p, h.total, 22) != h.crc) return LWF_ERR_OGG;
        OggStreamState &st = state(h.serial);
        const bool bos = h.htype & 2, eos = h.htype & 4, continued = h.htype & 1;
        if (!continued) { st.partial.clear(); st.in_packet = false; }
        const uint8_t *bp = p + 27 + h.nseg;
        const size_t q0 = queue.size();
        bool first_in_page = true;
        bool dropping = st.drop_continued && continued;
        st.drop_continued = false;
        for (size_t i = 0; i < h.nseg; i++) {
            const uint8_t l = p[27 + i];
            if (dropping) {                    // still inside the packet that began before the seek target
                bp += l;
                if (l < 255) dropping = false;
                continue;
            }
            st.partial.insert(st.partial.end(), bp, bp + l);
            st.in_packet = true;
            bp += l;
            if (l < 255) {
                Pending pk;
                pk.data.swap(st.partial);
                pk.serial = h.serial;
                pk.absgp = h.absgp;
                pk.first_stream = bos && first_in_page && !st.seen;
                pk.last_stream = false;
                pk.first_page = first_in_page;
                pk.last_page = false;
                queue.push_back(std::move(pk));
                st.partial.clear();
                st.in_packet = false;
                first_in_page = false;
                st.seen = true;
            }
        }
        if (queue.size() > q0) {
            queue.back().last_page = true;
            if (eos) queue.back().last_stream = true;
        }
        at += h.total;
        return LWB_OK;
    }

    // Page-granular seek inside logical stream `serial` (what ogg 0.8.0's PacketReader::seek_absgp gives
    // inside_ogg.rs:307-313): the read position moves to the start of the LAST page at or after byte offset `from`
    // whose granule position is <= goal (the first such page of the stream if none is), so that whatever is decoded
    // next lies at or before `goal`.  Pages are walked linearly: the data is a memory buffer.
    int seek_absgp(uint32_t serial, uint64_t goal, size_t from)
    {
        size_t pos = from, best = (size_t)-1, first = (size_t)-1;
        while (pos + 27 <= len) {
            PageHead h;
            if (page_head(pos, &h)) return LWF_ERR_OGG;
            if (h.serial == serial) {
                if (first == (size_t)-1) first = pos;
                if (h.absgp != ~0ull && h.absgp <= goal) best = pos;       // (-1: no packet finishes on this page)
                else if (h.absgp != ~0ull && h.absgp > goal) break;
            }
            pos += h.total;
        }
        if (first == (size_t)-1) return LWF_ERR_OGG;
        at = best != (size_t)-1 ? best : first;
        queue.clear();
        qhead = 0;
        OggStreamState &st = state(serial);
        st.partial.clear();
        st.in_packet = false;
        st.drop_continued = true;
        return LWB_OK;
    }

    int next(lwf_ogg_packet *out)
    {
        while (qhead >= queue.size()) {
            queue.clear();
            qhead = 0;
            const int rc = read_page();
            if (rc) return rc;
        }
        Pending &pk = queue[qhead++];
        current.swap(pk.data);
        out->data = current.data();
        out->len = current.size();
        out->stream_serial = pk.serial;
        out->absgp_page = pk.absgp;
        out->first_in_stream = pk.first_stream;
        out->last_in_stream = pk.last_stream;
        out->first_in_page = pk.first_page;
        out->last_in_page = pk.last_page;
        return LWB_OK;
    }
};

}  // namespace lwf

// ---------------------------------------------------------------------------------------------
// C ABI.  Nothing may unwind across it (lwfb::guarded): allocation failures become LWB_ERR_BUFFER.
// ---------------------------------------------------------------------------------------------
using lwfb::guarded;

// setup_of: headers that only hold an ident header and comments (lwfb::headers_sharing), whose codebooks, floors, residues,
// mappings and modes are those of setup_of; body() is what every use but the comments reads.
struct lwf_headers {
    lwf::Headers h;
    const lwf_headers *setup_of = nullptr;
    const lwf::Headers &body() const { return setup_of ? setup_of->h : h; }
};
struct lwf_ogg { lwf::Ogg o; };

extern "C" int lwf_headers_parse(const uint8_t *ident, size_t ident_len, const uint8_t *comment, size_t comment_len,
                                 const uint8_t *setup, size_t setup_len, lwf_headers **out)
{
    if (!ident || !comment || !setup || !out) return LWB_ERR_INVALID;
    return guarded([&]() -> int {
        std::unique_ptr<lwf_headers> h(new (std::nothrow) lwf_headers());
        if (!h) return LWB_ERR_BUFFER;
        int rc;
        if ((rc = lwf::read_ident(ident, ident_len, &h->h.ident))) return rc;
        if ((rc = lwf::read_comment(comment, comment_len, &h->h))) return rc;
        if ((rc = lwf::read_setup(setup, setup_len, &h->h))) return rc;
        *out = h.release();
        return LWB_OK;
    });
}

extern "C" void lwf_headers_destroy(lwf_headers *h) { delete h; }

extern "C" int lwf_headers_info(const lwf_headers *h, lwf_info *out)
{
    if (!h || !out) return LWB_ERR_INVALID;
    const lwf::Headers &s = h->body();
    out->audio_channels = s.ident.audio_channels;
    out->blocksize_0 = s.ident.blocksize_0;
    out->blocksize_1 = s.ident.blocksize_1;
    out->audio_sample_rate = s.ident.audio_sample_rate;
    out->bitrate_maximum = s.ident.bitrate_maximum;
    out->bitrate_nominal = s.ident.bitrate_nominal;
    out->bitrate_minimum = s.ident.bitrate_minimum;
    out->n_codebooks = (uint32_t)s.codebooks.size();
    out->n_floors = (uint32_t)s.floors.size();
    out->n_residues = (uint32_t)s.residues.size();
    out->n_mappings = (uint32_t)s.mappings.size();
    out->n_modes = (uint32_t)s.modes.size();
    out->n_comments = (uint32_t)h->h.comments.size();
    return LWB_OK;
}

extern "C" size_t lwf_headers_comment(const lwf_headers *h, int index, char *buf, size_t cap)
{
    if (!h) return 0;
    try {
        std::string s;
        if (index < 0) s = h->h.vendor;
        else if ((size_t)index < h->h.comments.size()) s = h->h.comments[index].first + "=" + h->h.comments[index].second;
        if (buf && cap) {
            const size_t k = std::min(cap - 1, s.size());
            std::memcpy(buf, s.data(), k);
            buf[k] = 0;
        }
        return s.size();
    } catch (...) {                  // nothing may unwind across the C ABI
        if (buf && cap) buf[0] = 0;
        return 0;
    }
}

extern "C" int lwf_headers_make_setup(const lwf_headers *h, lwb_ctx *ctx, lwb_setup **out)
{
    if (!h || !ctx || !out) return LWB_ERR_INVALID;
    return guarded([&]() -> int {
    const lwf::Headers &s = h->body();
    std::vector<lwb_floor_desc> floors(s.floors.size());
    for (size_t i = 0; i < s.floors.size(); i++) {
        std::memset(&floors[i], 0, sizeof(lwb_floor_desc));
        if (s.floors[i].type == 0) {
            floors[i].floor_type = LWB_FLOOR_TYPE_ZERO;
        } else {
            const lwf::Floor1 &f = s.floors[i].f1;
            floors[i].floor_type = LWB_FLOOR_TYPE_ONE;
            floors[i].floor1_multiplier = f.multiplier;
            floors[i].floor1_values = (uint8_t)f.x_list.size();
            for (size_t k = 0; k < f.x_list.size(); k++) floors[i].floor1_x_list[k] = f.x_list[k];
        }
    }
    std::vector<lwb_mapping_desc> maps(s.mappings.size());
    for (size_t i = 0; i < s.mappings.size(); i++) {
        const lwf::Mapping &m = s.mappings[i];
        std::memset(&maps[i], 0, sizeof(lwb_mapping_desc));
        maps[i].coupling_steps = (uint16_t)m.magnitudes.size();
        maps[i].submaps = (uint8_t)m.submap_floors.size();
        for (size_t k = 0; k < m.magnitudes.size(); k++) { maps[i].magnitudes[k] = m.magnitudes[k]; maps[i].angles[k] = m.angles[k]; }
        for (size_t k = 0; k < m.mux.size(); k++) maps[i].mux[k] = m.mux[k];
        for (size_t k = 0; k < m.submap_floors.size(); k++) maps[i].submap_floors[k] = m.submap_floors[k];
    }
    std::vector<lwb_mode_desc> modes(s.modes.size());
    for (size_t i = 0; i < s.modes.size(); i++) { modes[i].blockflag = s.modes[i].blockflag; modes[i].mapping = s.modes[i].mapping; }
    lwb_setup_desc d;
    std::memset(&d, 0, sizeof(d));
    d.audio_channels = s.ident.audio_channels;
    d.blocksize_0 = s.ident.blocksize_0;
    d.blocksize_1 = s.ident.blocksize_1;
    d.n_floors = (uint32_t)floors.size();
    d.floors = floors.data();
    d.n_mappings = (uint32_t)maps.size();
    d.mappings = maps.data();
    d.n_modes = (uint32_t)modes.size();
    d.modes = modes.data();
    // LWB_ENTRY_VQ: the codebooks' value tables (codebook_vq_lookup_vec) and the residues' partition sizes
    std::vector<lwb_codebook_desc> books(s.codebooks.size());
    for (size_t i = 0; i < s.codebooks.size(); i++) {
        const lwf::Codebook &cb = s.codebooks[i];
        books[i].dimensions = cb.dimensions;
        books[i].reserved = 0;
        books[i].entries = cb.dimensions ? (uint32_t)(cb.vq.size() / cb.dimensions) : 0;
        books[i].vq = cb.has_vq && !cb.vq.empty() ? cb.vq.data() : nullptr;
    }
    std::vector<lwb_residue_desc> resids(s.residues.size());
    for (size_t i = 0; i < s.residues.size(); i++) {
        std::memset(&resids[i], 0, sizeof(resids[i]));
        resids[i].residue_type = s.residues[i].type;
        resids[i].partition_size = s.residues[i].partition_size;
    }
    if (books.size() <= 256 && resids.size() <= 64) {
        d.n_codebooks = (uint32_t)books.size();
        d.codebooks = books.data();
        d.n_residues = (uint32_t)resids.size();
        d.residues = resids.data();
    }
    return lwb_setup_create(ctx, &d, out);
    });
}

// What LWB_ENTRY_VQ needs from a stream: <= 8 channels, and every VQ book a residue uses has a dimension that divides
// the residue's partition size (then the vectors of one pass never overlap and the device may add them in parallel).
extern "C" int lwf_headers_vq_capable(const lwf_headers *h)
{
    if (!h) return 0;
    const lwf::Headers &s = h->body();
    if (s.ident.audio_channels > 8 || s.codebooks.size() > 256 || s.residues.size() > 64) return 0;
    if ((size_t)s.ident.audio_channels << (s.ident.blocksize_1 - 1) > 12288) return 0;       // the device accumulators
    for (const lwf::Residue &r : s.residues)
        for (const lwf::ResidueBook &rb : r.books)
            for (int p = 0; p < 8; p++)
                if (rb.vals_used & (1u << p)) {
                    if (rb.val[p] >= s.codebooks.size()) return 0;
                    const lwf::Codebook &cb = s.codebooks[rb.val[p]];
                    if (!cb.has_vq || cb.dimensions == 0 || r.partition_size % cb.dimensions) return 0;
                    if (cb.vq.size() / cb.dimensions > 65536) return 0;                        // entries travel as u16
                }
    return 1;
}

// Whether decoding with `flags` can produce dense floor-0 curves (a type-0 floor that does not travel as a record).
static bool needs_dense(const lwf::Headers &h, int flags)
{
    for (const auto &fl : h.floors)
        if (fl.type == 0 && !((flags & LWF_DECODE_FLOOR0_RECORDS) && lwf::floor0_record_ok(fl.f0))) return true;
    return false;
}

// The lwb_setup_set_floor0 descriptions of the headers' type-0 floors that can travel as records (floor index, desc; the
// tables point into the headers).  lwf_headers_make_setup_floor0 (lwb_api.cu) applies them.
namespace lwf {
void floor0_descs(const lwf_headers *h, std::vector<uint32_t> *index, std::vector<lwb_floor0_desc> *descs)
{
    for (size_t i = 0; i < h->body().floors.size(); i++) {
        const Floor &fl = h->body().floors[i];
        if (fl.type != 0 || !floor0_record_ok(fl.f0)) continue;
        lwb_floor0_desc d;
        std::memset(&d, 0, sizeof(d));
        d.order = fl.f0.order;
        d.amplitude_bits = fl.f0.amplitude_bits;
        d.amplitude_offset = fl.f0.amplitude_offset;
        d.rate = fl.f0.rate;
        d.bark_map_size = fl.f0.bark_map_size;
        d.bark_cos_omega[0] = fl.f0.bark_cos_omega[0].data();      // the tables the dense path uses
        d.bark_cos_omega[1] = fl.f0.bark_cos_omega[1].data();
        index->push_back((uint32_t)i);
        descs->push_back(d);
    }
}
}  // namespace lwf

extern "C" int lwf_packet_decode_vq(const lwf_headers *h, const uint8_t *packet, size_t len, lwf_decoded_packet *out,
                                    lwb_vq_run *runs, size_t run_capacity, size_t *n_runs, uint16_t *entries, size_t entry_capacity,
                                    size_t *n_entries)
{
    return lwf_packet_decode_vq_ex(h, packet, len, out, runs, run_capacity, n_runs, entries, entry_capacity, n_entries, 0);
}

extern "C" int lwf_packet_decode_vq_ex(const lwf_headers *h, const uint8_t *packet, size_t len, lwf_decoded_packet *out,
                                       lwb_vq_run *runs, size_t run_capacity, size_t *n_runs, uint16_t *entries, size_t entry_capacity,
                                       size_t *n_entries, int flags)
{
    if (!h || (!packet && len) || !out || !out->floor_kind || !out->floor1_y || (!runs && run_capacity) || (!entries && entry_capacity) ||
        !n_runs || !n_entries || (flags & ~LWF_DECODE_FLOOR0_RECORDS))
        return LWB_ERR_INVALID;
    if (!out->dense_floor && needs_dense(h->body(), flags)) return LWB_ERR_INVALID;
    *n_runs = *n_entries = 0;
    return guarded([&]() -> int {
        lwf::VqSink sink;
        sink.runs = runs;
        sink.run_cap = run_capacity;
        sink.entries = entries;
        sink.ent_cap = entry_capacity;
        const int rc = lwf::packet_decode(h->body(), packet, len, out, &sink, (flags & LWF_DECODE_FLOOR0_RECORDS) != 0);
        if (rc) return rc;
        if (sink.overflow) return LWB_ERR_BUFFER;
        *n_runs = sink.n_runs;
        *n_entries = sink.n_ent;
        return LWB_OK;
    });
}

extern "C" int lwf_packet_decode(const lwf_headers *h, const uint8_t *packet, size_t len, lwf_decoded_packet *out)
{
    return lwf_packet_decode_ex(h, packet, len, out, 0);
}

extern "C" int lwf_packet_decode_ex(const lwf_headers *h, const uint8_t *packet, size_t len, lwf_decoded_packet *out, int flags)
{
    if (!h || (!packet && len) || !out || !out->floor_kind || !out->floor1_y || !out->residue || (flags & ~LWF_DECODE_FLOOR0_RECORDS))
        return LWB_ERR_INVALID;
    if (!out->dense_floor && needs_dense(h->body(), flags)) return LWB_ERR_INVALID;
    return guarded([&] { return lwf::packet_decode(h->body(), packet, len, out, nullptr, (flags & LWF_DECODE_FLOOR0_RECORDS) != 0); });
}

// get_decoded_sample_count, audio.rs:874-909
extern "C" int lwf_decoded_sample_count(const lwf_headers *h, const uint8_t *packet, size_t len, size_t *n_samples)
{
    if (!h || (!packet && len) || !n_samples) return LWB_ERR_INVALID;
    lwf::BitReader rdr(packet, len);
    lwf::PacketHead ph;
    const int rc = lwf::packet_head(h->body(), rdr, &ph);
    if (rc) return rc;
    const uint32_t n = ph.n, n0 = 1u << h->body().ident.blocksize_0;
    const uint32_t ls = ph.prev ? 0 : (n - n0) >> 2;
    const uint32_t rs = ph.next ? n >> 1 : (n * 3 - n0) >> 2;
    *n_samples = rs - ls;
    return LWB_OK;
}

extern "C" int lwf_ogg_open(const uint8_t *data, size_t len, lwf_ogg **out)
{
    if ((!data && len) || !out) return LWB_ERR_INVALID;
    lwf_ogg *o = new (std::nothrow) lwf_ogg();
    if (!o) return LWB_ERR_BUFFER;
    o->o.d = data;
    o->o.len = len;
    *out = o;
    return LWB_OK;
}
extern "C" void lwf_ogg_close(lwf_ogg *o) { delete o; }
extern "C" int lwf_ogg_next_packet(lwf_ogg *o, lwf_ogg_packet *pkt)
{
    if (!o || !pkt) return LWB_ERR_INVALID;
    return guarded([&] { return o->o.next(pkt); });
}

// ---------------------------------------------------------------------------------------------
// OggStreamReader, inside_ogg.rs:60-227
// ---------------------------------------------------------------------------------------------
struct lwf_reader {
    lwb_ctx *ctx = nullptr;
    lwf_ogg *ogg = nullptr;
    lwf_headers *hdr = nullptr;
    lwb_setup *setup = nullptr;
    lwb_stream *pwr = nullptr;
    uint32_t serial = 0;
    lwfb::Granule gp;
    size_t audio_start = 0;        // byte offset of the first page after the current stream's headers
    lwfb::PacketScratch pkt;
    std::vector<float> dropped;    // the PCM of packets decoded and dropped
};

static void reader_drop_stream(lwf_reader *r)
{
    if (r->pwr) lwb_stream_destroy(r->pwr);
    if (r->setup) lwb_setup_destroy(r->setup);
    if (r->hdr) lwf_headers_destroy(r->hdr);
    r->pwr = nullptr;
    r->setup = nullptr;
    r->hdr = nullptr;
}

// read_headers, inside_ogg.rs:19-39 (`first`: the ident packet has already been read)
static int reader_read_headers(lwf_reader *r, const lwf_ogg_packet *first)
{
    lwfb::HeaderPackets hp;
    if (first) hp.ident.assign(first->data, first->data + first->len);
    int rc = lwfb::read_header_packets(r->ogg, first != nullptr, hp);
    if (rc) return rc;
    lwf_headers *h = nullptr;
    if ((rc = lwf_headers_parse(hp.ident.data(), hp.ident.size(), hp.comment.data(), hp.comment.size(), hp.setup.data, hp.setup.len, &h)))
        return rc;
    reader_drop_stream(r);
    r->hdr = h;
    if ((rc = lwf_headers_make_setup(h, r->ctx, &r->setup))) return rc;
    if ((rc = lwb_stream_open(r->ctx, r->setup, &r->pwr))) return rc;
    r->serial = hp.serial;
    r->gp.has = false;
    r->audio_start = lwfb::pager_offset(r->ogg);
    r->pkt = lwfb::PacketScratch(h);
    return LWB_OK;
}

extern "C" int lwf_reader_open(lwb_ctx *ctx, const uint8_t *data, size_t len, lwf_reader **out)
{
    if (!ctx || (!data && len) || !out) return LWB_ERR_INVALID;
    std::unique_ptr<lwf_reader> r(new (std::nothrow) lwf_reader());
    if (!r) return LWB_ERR_BUFFER;
    r->ctx = ctx;
    int rc = lwf_ogg_open(data, len, &r->ogg);
    if (rc) return rc;
    if ((rc = guarded([&] { return reader_read_headers(r.get(), nullptr); }))) {
        reader_drop_stream(r.get());
        lwf_ogg_close(r->ogg);
        return rc;
    }
    *out = r.release();
    return LWB_OK;
}

extern "C" void lwf_reader_close(lwf_reader *r)
{
    if (!r) return;
    reader_drop_stream(r);
    lwf_ogg_close(r->ogg);
    delete r;
}

extern "C" const lwf_headers *lwf_reader_headers(const lwf_reader *r) { return r ? r->hdr : nullptr; }

// read_audio_packet_generic through the CUDA back half
static int reader_decode(lwf_reader *r, const lwf_ogg_packet &pk, int out_format, void *out, size_t cap, size_t *n)
{
    lwf_decoded_packet dp = r->pkt.packet();
    int rc = lwf_packet_decode(r->hdr, pk.data, pk.len, &dp);
    if (rc) return rc;
    lwb_packet p;
    std::memset(&p, 0, sizeof(p));
    p.mode_number = dp.mode_number;
    p.prev_window_flag = dp.prev_window_flag;
    p.next_window_flag = dp.next_window_flag;
    p.floor_kind = dp.floor_kind;
    p.floor1_y = dp.floor1_y;
    p.dense_floor = dp.dense_floor;
    p.residue = dp.residue;
    return lwb_decode_packet(r->pwr, &p, out_format, out, cap, n);
}

// Decodes pk on the reader's stream state and drops its PCM
static int reader_decode_drop(lwf_reader *r, const lwf_ogg_packet &pk)
{
    const size_t C = r->hdr->h.ident.audio_channels, n1 = (size_t)1 << r->hdr->h.ident.blocksize_1;
    r->dropped.resize(C * n1);
    size_t n = 0;
    return reader_decode(r, pk, LWB_OUT_F32_PLANAR, r->dropped.data(), n1, &n);
}

// read_next_audio_packet, inside_ogg.rs:107-143
static int reader_next_audio_packet(lwf_reader *r, lwf_ogg_packet *pk)
{
    int rc = lwfb::next_packet_of(r->ogg, r->serial, pk, nullptr);
    if (rc || pk->stream_serial == r->serial) return rc;
    // a chained stream begins: new headers, new state; its first audio packet is decoded and dropped
    if ((rc = reader_read_headers(r, pk))) return rc;
    if ((rc = lwf_ogg_next_packet(r->ogg, pk))) return rc;
    if ((rc = reader_decode_drop(r, *pk))) return rc;
    r->gp = lwfb::Granule{true, pk->absgp_page};
    return lwf_ogg_next_packet(r->ogg, pk);
}

// dec_packet_generic, inside_ogg.rs:207-229: decode, truncate at the end of the stream, account the granule position
static int reader_dec_packet(lwf_reader *r, const lwf_ogg_packet &pk, int out_format, void *out, size_t cap_total, size_t *n_samples)
{
    size_t n = 0;
    const size_t cap = cap_total / r->hdr->h.ident.audio_channels;
    int rc = reader_decode(r, pk, out_format, out, cap, &n);
    if (rc) return rc;
    n = r->gp.cut(pk, n);
    r->gp.step(pk, n);
    *n_samples = n;
    return LWB_OK;
}

// read_dec_packet_generic, inside_ogg.rs:191-205
extern "C" int lwf_reader_read_dec_packet(lwf_reader *r, int out_format, void *out, size_t cap_total, size_t *n_samples)
{
    if (!r || !out || !n_samples) return LWB_ERR_INVALID;
    *n_samples = 0;
    return guarded([&] {
        lwf_ogg_packet pk;
        int rc = reader_next_audio_packet(r, &pk);
        if (rc) return rc;
        return reader_dec_packet(r, pk, out_format, out, cap_total, n_samples);
    });
}

// skip_samples_linear, inside_ogg.rs:244-283: packets are only measured (get_decoded_sample_count) until the one that
// holds the target; the packet before it is decoded on a fresh PreviousWindowRight (and dropped) so that the target
// packet overlaps with the right history, then the target packet is decoded and returned.
extern "C" int lwf_reader_skip_samples_linear(lwf_reader *r, size_t to_skip, int out_format, void *out, size_t cap_total,
                                              size_t *n_samples, size_t *left_to_skip, int *got_packet)
{
    if (!r || !out || !n_samples || !left_to_skip || !got_packet) return LWB_ERR_INVALID;
    *n_samples = 0;
    *got_packet = 0;
    *left_to_skip = to_skip;
    return guarded([&]() -> int {
        std::vector<uint8_t> last;             // Option<Packet>: the packet read before `next`
        lwf_ogg_packet last_pk;
        std::memset(&last_pk, 0, sizeof(last_pk));
        lwfb::SkipWalk walk;
        walk.to_skip = to_skip;
        for (;;) {
            lwf_ogg_packet next;
            int rc = reader_next_audio_packet(r, &next);
            if (rc == LWF_ERR_NO_MORE_PACKETS) { *left_to_skip = walk.to_skip; return LWB_OK; }      // Ok((None, to_skip))
            if (rc) return rc;
            size_t cnt = 0;
            if ((rc = lwf_decoded_sample_count(r->hdr, next.data, next.len, &cnt))) return rc;
            if (walk.target(r->gp, next, cnt)) {                  // :263-271
                if (walk.have_last) {
                    lwb_stream_reset(r->pwr);
                    last_pk.data = last.data();
                    last_pk.len = last.size();
                    // `next.data` points into the pager's current buffer, which stays valid: nothing is read in between
                    if ((rc = reader_decode_drop(r, last_pk))) return rc;
                }
                if ((rc = reader_dec_packet(r, next, out_format, out, cap_total, n_samples))) return rc;
                *got_packet = 1;
                *left_to_skip = walk.to_skip;
                return LWB_OK;
            }
            last.assign(next.data, next.data + next.len);
            last_pk = next;
        }
    });
}

// seek_absgp_pg, inside_ogg.rs:307-313: page-granular seek, then cur_absgp = None and a fresh PreviousWindowRight
extern "C" int lwf_reader_seek_absgp_pg(lwf_reader *r, uint64_t absgp)
{
    if (!r) return LWB_ERR_INVALID;
    return guarded([&] {
        const int rc = lwfb::pager_seek(r->ogg, r->serial, absgp, r->audio_start);
        if (rc) return rc;
        r->gp.has = false;
        return lwb_stream_reset(r->pwr);
    });
}

extern "C" int lwf_reader_last_absgp(const lwf_reader *r, uint64_t *absgp)
{
    if (!r || !absgp) return LWB_ERR_INVALID;
    if (!r->gp.has) return 1;
    *absgp = r->gp.absgp;
    return 0;
}

// ---------------------------------------------------------------------------------------------
// lwf_batcher: parallel host entropy decode + one batched synthesis call
// ---------------------------------------------------------------------------------------------
using namespace lwfb;

extern "C" int lwf_batcher_create(lwb_ctx *ctx, const lwf_headers *h, int threads, lwf_batcher **out)
{
    if (!ctx || !h || !out) return LWB_ERR_INVALID;
    return guarded([&]() -> int {
        std::unique_ptr<lwf_batcher> b(new lwf_batcher());
        b->ctx = ctx;
        if (threads <= 0) threads = (int)std::thread::hardware_concurrency();
        b->threads = std::max(1, threads);
        b->groups.emplace_back(new Group());
        Group &g = *b->groups[0];
        g.channels = h->body().ident.audio_channels;
        g.bs0 = h->body().ident.blocksize_0;
        g.bs1 = h->body().ident.blocksize_1;
        b->sets.push_back(HeaderSet{h, nullptr, 0});
        update_floor0(b.get());
        *out = b.release();
        return LWB_OK;
    });
}

extern "C" void lwf_batcher_destroy(lwf_batcher *b)
{
    if (!b) return;
    if (b->release) b->release(b, true);                // the arenas may still be read by submitted batches
    delete b;
}

extern "C" int lwf_batcher_set_entry(lwf_batcher *b, int entry)
{
    if (!b || (entry != LWB_ENTRY_RESIDUE && entry != LWB_ENTRY_VQ)) return LWB_ERR_INVALID;
    if (entry == LWB_ENTRY_VQ)
        for (const HeaderSet &s : b->sets)
            if (!lwf_headers_vq_capable(s.h)) return LWB_ERR_INVALID;
    b->entry = entry;
    return LWB_OK;
}

extern "C" uint64_t lwf_batcher_last_input_bytes(const lwf_batcher *b) { return b ? b->in_bytes : 0; }

extern "C" int lwf_batcher_set_floor0(lwf_batcher *b, int records)
{
    if (!b) return LWB_ERR_INVALID;
    b->floor0_records = records != 0;
    update_floor0(b);
    return LWB_OK;
}

extern "C" void lwf_batcher_last_timing(const lwf_batcher *b, double *e, double *s)
{
    if (!b) return;
    if (e) *e = b->t_entropy;
    if (s) *s = b->t_synth;
}

namespace lwfb {
double now_s()
{
    return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

int run_pool(int threads, size_t n, const std::function<void(size_t k, int w)> &item)
{
    const int nt = (int)std::min<size_t>((size_t)std::max(1, threads), std::max<size_t>(1, n));
    std::atomic<size_t> next(0);
    std::atomic<bool> failed(false);
    auto worker = [&](int w) {
        try {
            for (size_t k; (k = next.fetch_add(1)) < n;) item(k, w);
        } catch (...) {
            failed.store(true);
        }
    };
    std::vector<std::thread> pool;
    try {
        pool.reserve((size_t)nt);
        for (int t = 1; t < nt; t++) pool.emplace_back(worker, t);
    } catch (...) {
        // no more threads to be had (std::system_error) or no memory for the vector: go on with the workers that did
        // start -- they share the item counter, so the work is the same -- instead of unwinding past joinable threads
    }
    worker(0);
    for (auto &t : pool) t.join();
    return failed.load() ? LWB_ERR_BUFFER : LWB_OK;
}

PacketScratch::PacketScratch(const lwf_headers *h)
    : kinds(h->body().ident.audio_channels), ys(kinds.size() * LWB_MAX_POSTS),
      dense(kinds.size() << (h->body().ident.blocksize_1 - 1)), residue(dense.size())
{
}

lwf_decoded_packet PacketScratch::packet()
{
    lwf_decoded_packet dp;
    std::memset(&dp, 0, sizeof(dp));
    dp.floor_kind = kinds.data();
    dp.floor1_y = ys.data();
    dp.dense_floor = dense.data();
    dp.residue = residue.data();
    return dp;
}

lwf_ogg *ogg_clone(const lwf_ogg *o)
{
    try {
        return new lwf_ogg(*o);
    } catch (...) {
        return nullptr;
    }
}

int headers_sharing(const lwf_headers *shared, const uint8_t *comment, size_t comment_len, lwf_headers **out)
{
    if (!comment && comment_len) return LWB_ERR_INVALID;
    return guarded([&]() -> int {
        std::unique_ptr<lwf_headers> h(new lwf_headers());
        const int rc = lwf::read_comment(comment, comment_len, &h->h);
        if (rc) return rc;
        h->h.ident = shared->body().ident;
        h->setup_of = shared->setup_of ? shared->setup_of : shared;
        *out = h.release();
        return LWB_OK;
    });
}

size_t Granule::cut(const lwf_ogg_packet &pk, size_t n) const
{
    if (!has || !pk.last_in_stream) return n;
    const uint64_t target = pk.absgp_page > absgp ? pk.absgp_page - absgp : 0;
    return target < n ? (size_t)target : n;
}

void Granule::step(const lwf_ogg_packet &pk, size_t n)
{
    if (pk.last_in_page) {
        has = true;
        absgp = pk.absgp_page;
    } else if (has) {
        absgp += n;
    }
}

bool SkipWalk::target(Granule &gp, const lwf_ogg_packet &pk, size_t n)
{
    if (gp.has && pk.last_in_stream) have_last = false;
    n = gp.cut(pk, n);
    if (to_skip < n) return true;
    to_skip -= n;
    if (gp.has) gp.absgp += n;
    have_last = true;
    return false;
}

size_t pager_offset(const lwf_ogg *o) { return o->o.at; }

int pager_seek(lwf_ogg *o, uint32_t serial, uint64_t absgp, size_t from) { return o->o.seek_absgp(serial, absgp, from); }

int read_header_packets(lwf_ogg *o, bool chained, HeaderPackets &hp)
{
    lwf_ogg_packet &pk = hp.setup;
    auto next = [&]() {
        const int rc = lwf_ogg_next_packet(o, &pk);
        return rc == LWF_ERR_NO_MORE_PACKETS ? (int)LWF_ERR_OGG : rc;
    };
    int rc;
    if (!chained) {
        if ((rc = next())) return rc;
        hp.ident.assign(pk.data, pk.data + pk.len);
        hp.serial = pk.stream_serial;
    }
    do {
        if ((rc = next())) return rc;
    } while (!chained && pk.stream_serial != hp.serial);
    hp.comment.assign(pk.data, pk.data + pk.len);
    do {
        if ((rc = next())) return rc;
    } while (!chained && pk.stream_serial != hp.serial);
    hp.serial = pk.stream_serial;
    return LWB_OK;
}

int next_packet_of(lwf_ogg *o, uint32_t serial, lwf_ogg_packet *pk, size_t *reads)
{
    for (;;) {
        if (reads) ++*reads;
        const int rc = lwf_ogg_next_packet(o, pk);
        if (rc || pk->stream_serial == serial || pk->first_in_stream) return rc;
    }
}

void assign_sets(const lwf_batcher *b, const lwf_stream_job *jobs, size_t n_jobs, std::vector<JobPlan> &plan)
{
    for (size_t j = 0; j < n_jobs; j++) plan[j].set = b->set_of ? b->set_of(b, jobs[j].stream) : 0;
}

void update_floor0(lwf_batcher *b)
{
    for (auto &g : b->groups) g->has_floor0 = false;
    for (const HeaderSet &s : b->sets)
        if (needs_dense(s.h->body(), b->floor0_records ? LWF_DECODE_FLOOR0_RECORDS : 0)) b->groups[s.group]->has_floor0 = true;
}

// entropy decode of jobs list[0 .. n) into arena set `set` of their groups on the batcher's host threads
int batch_entropy(lwf_batcher *b, size_t set, lwf_stream_job *jobs, const size_t *list, size_t n, std::vector<JobPlan> &plan,
                  std::vector<uint32_t> &decoded, std::vector<int32_t> &dec_status, std::vector<size_t> *used)
{
    const size_t n_groups = b->groups.size();
    // pass 1 (cheap, serial): packet headers -> blocksizes -> arena offsets in the job's group.  A packet whose header
    // cannot be read ends its stream's chain there (its error is reported after the earlier ones ran).
    std::vector<uint64_t> coeff_total(n_groups, 0), pkt_total(n_groups, 0);
    std::vector<std::vector<size_t>> members(n_groups);        // the jobs of each group, in list order
    for (size_t i = 0; i < n; i++) {
        const size_t j = list[i];
        const lwf_stream_job &job = jobs[j];
        JobPlan &p = plan[j];
        const size_t g = b->sets[p.set].group;
        const lwf::Headers &H = b->sets[p.set].h->body();
        const size_t C = b->groups[g]->channels;
        p.coeff0 = coeff_total[g];
        p.pkt0 = pkt_total[g];
        p.usable = 0;
        p.head_status = LWB_OK;
        p.slot = members[g].size();
        members[g].push_back(j);
        for (uint32_t k = 0; k < job.n_packets; k++) {
            lwf::BitReader rdr(job.packets[k], job.lengths[k]);
            lwf::PacketHead ph;
            const int rc = lwf::packet_head(H, rdr, &ph);
            if (rc) { p.head_status = rc; break; }
            coeff_total[g] += (uint64_t)C * (ph.n / 2);
            p.usable++;
        }
        pkt_total[g] += p.usable;
    }
    used->clear();
    for (size_t g = 0; g < n_groups; g++)
        if (!members[g].empty()) used->push_back(g);
    if (used->empty()) used->push_back(0);
    const bool vq = b->entry == LWB_ENTRY_VQ;
    for (size_t g : *used) {
        BatchArena &ar = b->groups[g]->arena[set];
        const size_t rows = (size_t)pkt_total[g] * b->groups[g]->channels;
        if ((!vq && !ar.coeffs.ensure((size_t)coeff_total[g] * 4 + 16)) || !ar.kinds.ensure(rows + 16) || !ar.ys.ensure(rows * LWB_MAX_POSTS * 4 + 16) ||
            (b->groups[g]->has_floor0 && !ar.dense.ensure((size_t)coeff_total[g] * 4 + 16)) ||
            (vq && (!ar.vqroff.ensure(((size_t)pkt_total[g] + 1) * 8 + 16) || !ar.vqeoff.ensure(((size_t)pkt_total[g] + 1) * 8 + 16))))
            return LWB_ERR_BUFFER;
        // VQ: every stream's records are collected per job first (their number is only known after the decode), then
        // packed into one pinned arena with per-packet offsets
        if (vq) {
            const size_t m = members[g].size();
            if (ar.job_runs.size() < m) { ar.job_runs.resize(m); ar.job_ents.resize(m); }
            for (size_t s = 0; s < m; s++) { ar.job_runs[s].clear(); ar.job_ents[s].clear(); }
        }
        ar.modes.resize(pkt_total[g]);
        ar.prevs.resize(pkt_total[g]);
        ar.nexts.resize(pkt_total[g]);
    }
    // pass 2 (parallel over all jobs of the list): entropy decode straight into the arenas of each job's group
    std::vector<std::vector<lwb_vq_run>> scratch_runs(vq ? b->threads : 0);    // LWB_ENTRY_VQ: one packet's records
    std::vector<std::vector<uint16_t>> scratch_ents(scratch_runs.size());       // (see below), per worker
    auto decode = [&](size_t i, int w) {
        const size_t j = list[i];
        const lwf_stream_job &job = jobs[j];
        const JobPlan &p = plan[j];
        const lwf::Headers &H = b->sets[p.set].h->body();
        Group &G = *b->groups[b->sets[p.set].group];
        BatchArena &ar = G.arena[set];
        const size_t C = G.channels;
        float *coeffs = (float *)ar.coeffs.p, *dense = G.has_floor0 ? (float *)ar.dense.p : nullptr;
        uint8_t *kinds = (uint8_t *)ar.kinds.p;
        uint32_t *ys = (uint32_t *)ar.ys.p;
        uint64_t *run_off = vq ? (uint64_t *)ar.vqroff.p : nullptr, *ent_off = vq ? (uint64_t *)ar.vqeoff.p : nullptr;
        uint64_t coff = p.coeff0;
        for (uint32_t k = 0; k < p.usable; k++) {
            const uint64_t pi = p.pkt0 + k;
            lwf_decoded_packet dp;
            std::memset(&dp, 0, sizeof(dp));
            dp.floor_kind = kinds + pi * C;
            dp.floor1_y = ys + pi * C * LWB_MAX_POSTS;
            dp.residue = vq ? nullptr : coeffs + coff;
            dp.dense_floor = dense ? dense + coff : nullptr;
            int rc;
            if (vq) {
                std::vector<lwb_vq_run> &jr = ar.job_runs[p.slot];
                std::vector<uint16_t> &je = ar.job_ents[p.slot];
                std::vector<lwb_vq_run> &runs = scratch_runs[w];
                std::vector<uint16_t> &ents = scratch_ents[w];
                // decoded into the worker's scratch (a packet of b bytes holds fewer than 8 b codewords), then only what
                // it produced is appended (growing the job's vectors to the bound first meant zero-filling ~22 KB per
                // 280-byte packet)
                const size_t cap = (size_t)job.lengths[k] * 8 + 16;
                if (runs.size() < cap) { runs.resize(cap); ents.resize(cap); }
                lwf::VqSink sink;
                sink.runs = runs.data();
                sink.run_cap = cap;
                sink.entries = ents.data();
                sink.ent_cap = cap;
                rc = lwf::packet_decode(H, job.packets[k], job.lengths[k], &dp, &sink, b->floor0_records);
                if (!rc && sink.overflow) rc = LWB_ERR_BUFFER;
                if (!rc) {
                    jr.insert(jr.end(), runs.data(), runs.data() + sink.n_runs);
                    je.insert(je.end(), ents.data(), ents.data() + sink.n_ent);
                }
                run_off[pi + 1] = rc ? 0 : sink.n_runs;      // counts for now; turned into offsets below
                ent_off[pi + 1] = rc ? 0 : sink.n_ent;
            } else {
                rc = lwf::packet_decode(H, job.packets[k], job.lengths[k], &dp, nullptr, b->floor0_records);
            }
            if (rc) { dec_status[j] = rc; break; }
            ar.modes[pi] = dp.mode_number;
            ar.prevs[pi] = dp.prev_window_flag;
            ar.nexts[pi] = dp.next_window_flag;
            coff += (uint64_t)C * (dp.n / 2);
            decoded[j]++;
        }
    };
    if (const int rc = run_pool(b->threads, n, decode)) return rc;
    if (vq) {
        // counts -> offsets (rows of packets that were not decoded own nothing), then one packed copy of each array
        for (size_t g : *used) {
            BatchArena &ar = b->groups[g]->arena[set];
            uint64_t *run_off = (uint64_t *)ar.vqroff.p, *ent_off = (uint64_t *)ar.vqeoff.p;
            run_off[0] = ent_off[0] = 0;
            for (size_t j : members[g])
                for (uint32_t k = 0; k < plan[j].usable; k++) {
                    const uint64_t pi = plan[j].pkt0 + k;
                    const bool ok = k < decoded[j];
                    run_off[pi + 1] = run_off[pi] + (ok ? run_off[pi + 1] : 0);
                    ent_off[pi + 1] = ent_off[pi] + (ok ? ent_off[pi + 1] : 0);
                }
            if (!ar.vqrun.ensure((size_t)run_off[pkt_total[g]] * sizeof(lwb_vq_run) + 16) || !ar.vqent.ensure((size_t)ent_off[pkt_total[g]] * 2 + 16))
                return LWB_ERR_BUFFER;
        }
        // ~3 KB per stereo long packet: copied by the pool as well (one thread alone would take about as long over it as
        // the whole pool over the entropy decode)
        auto copy = [&](size_t i, int) {
            const JobPlan &p = plan[list[i]];
            BatchArena &ar = b->groups[b->sets[p.set].group]->arena[set];
            const std::vector<lwb_vq_run> &jr = ar.job_runs[p.slot];
            const std::vector<uint16_t> &je = ar.job_ents[p.slot];
            if (!jr.empty()) std::memcpy((lwb_vq_run *)ar.vqrun.p + ((uint64_t *)ar.vqroff.p)[p.pkt0], jr.data(), jr.size() * sizeof(lwb_vq_run));
            if (!je.empty()) std::memcpy((uint16_t *)ar.vqent.p + ((uint64_t *)ar.vqeoff.p)[p.pkt0], je.data(), je.size() * sizeof(uint16_t));
        };
        if (const int rc = run_pool(b->threads, n, copy)) return rc;
    }
    for (size_t g : *used) {
        BatchArena &ar = b->groups[g]->arena[set];
        const uint64_t rows = pkt_total[g] * b->groups[g]->channels, pk = pkt_total[g];
        // what crosses to the device: residues or VQ records, dense floor-0 curves, floor kinds and floor1_y rows
        ar.in_bytes = rows + rows * LWB_MAX_POSTS * 4 + (b->groups[g]->has_floor0 ? coeff_total[g] * 4 : 0) +
                      (vq ? (pk + 1) * 16 + ((uint64_t *)ar.vqroff.p)[pk] * sizeof(lwb_vq_run) + ((uint64_t *)ar.vqeoff.p)[pk] * 2 : coeff_total[g] * 4);
        ar.coeff_total = coeff_total[g];
        // the group's chains
        ar.job = members[g];
        ar.chains.assign(members[g].size(), lwb_chain());
        for (size_t s = 0; s < members[g].size(); s++) {
            const size_t j = members[g][s];
            lwb_chain &c = ar.chains[s];
            std::memset(&c, 0, sizeof(c));
            c.stream = jobs[j].stream;
            c.n_packets = decoded[j];
            c.mode_numbers = ar.modes.data() + plan[j].pkt0;
            c.prev_window_flags = ar.prevs.data() + plan[j].pkt0;
            c.next_window_flags = ar.nexts.data() + plan[j].pkt0;
            c.coeff_offset = plan[j].coeff0;
            c.packet_index = plan[j].pkt0;
            c.out_offset = jobs[j].out_offset;
            c.out_stride = jobs[j].out_stride;
        }
    }
    return LWB_OK;
}

lwb_batch_io batch_io(const lwf_batcher *b, size_t g, const BatchArena &ar, int out_format, void *pcm)
{
    lwb_batch_io io;
    std::memset(&io, 0, sizeof(io));
    io.entry = b->entry;
    io.memory = LWB_MEM_HOST;
    io.coeffs = (const float *)ar.coeffs.p;
    io.vq_runs = (const lwb_vq_run *)ar.vqrun.p;
    io.vq_run_offsets = (const uint64_t *)ar.vqroff.p;
    io.vq_entries = (const uint16_t *)ar.vqent.p;
    io.vq_entry_offsets = (const uint64_t *)ar.vqeoff.p;
    io.dense_floor = b->groups[g]->has_floor0 ? (const float *)ar.dense.p : nullptr;
    io.floor_kind = (const uint8_t *)ar.kinds.p;
    io.floor1_y = (const uint32_t *)ar.ys.p;
    io.out_format = out_format;
    io.pcm = pcm;
    return io;
}

// The synthesis's results, and where it ran every packet the entropy decode passed, the entropy or header error that
// stopped the stream there.
void job_results(lwf_stream_job *jobs, const BatchArena &ar, const std::vector<JobPlan> &plan, const std::vector<uint32_t> &decoded,
                 const std::vector<int32_t> &dec_status)
{
    for (size_t s = 0; s < ar.chains.size(); s++) {
        const lwb_chain &c = ar.chains[s];
        const size_t j = ar.job[s];
        jobs[j].n_samples = c.n_samples;
        jobs[j].packets_done = c.packets_done;
        jobs[j].status = c.status;
        if (c.status == LWB_OK && c.packets_done == decoded[j] && decoded[j] < jobs[j].n_packets)
            jobs[j].status = dec_status[j] != LWB_OK ? dec_status[j] : plan[j].head_status;
    }
}

int check_jobs(const lwf_stream_job *jobs, size_t n_jobs)
{
    for (size_t j = 0; j < n_jobs; j++)
        if (!jobs[j].stream || (jobs[j].n_packets && (!jobs[j].packets || !jobs[j].lengths))) return LWB_ERR_INVALID;
    return LWB_OK;
}
}  // namespace lwfb

extern "C" int lwf_batcher_decode(lwf_batcher *b, lwf_stream_job *jobs, size_t n_jobs, int out_format, void *pcm)
{
    if (!b || (!jobs && n_jobs) || !pcm || check_jobs(jobs, n_jobs)) return LWB_ERR_INVALID;
    return guarded([&] {
        int rc = b->release ? b->release(b, false) : LWB_OK;      // submitted batches may still read the arenas
        if (rc) return rc;
        std::vector<JobPlan> plan(n_jobs);
        std::vector<uint32_t> decoded(n_jobs, 0);
        std::vector<int32_t> dec_status(n_jobs, LWB_OK);
        assign_sets(b, jobs, n_jobs, plan);
        // Slices of streams: while the GPU call of slice i runs (on one helper thread -- an lwb_ctx takes
        // one caller at a time), the pool already entropy-decodes slice i + 1 into the other arena.  A slice holds the
        // jobs of one group (one batch); each group is cut into up to four slices, and the slices of all groups follow
        // each other through the pipeline.
        std::vector<std::vector<size_t>> members(b->groups.size());
        for (size_t j = 0; j < n_jobs; j++) members[b->sets[plan[j].set].group].push_back(j);
        std::vector<std::vector<size_t>> slices;
        for (size_t g = 0; g < members.size(); g++) {
            const size_t m = members[g].size();
            if (!m && (g || n_jobs)) continue;        // no jobs at all: one empty batch, as for any other job count
            const size_t n_slices = std::max<size_t>(1, std::min<size_t>(4, m / 8));
            for (size_t sl = 0; sl < n_slices; sl++)
                slices.emplace_back(members[g].begin() + m * sl / n_slices, members[g].begin() + m * (sl + 1) / n_slices);
        }
        double entropy_busy = 0, synth_busy = 0;
        uint64_t in_bytes = 0;
        int synth_rc = LWB_OK;
        std::vector<size_t> used;
        std::thread synth;
        struct Joiner { std::thread &t; ~Joiner() { if (t.joinable()) t.join(); } } joiner{synth};   // also on unwinding
        for (size_t sl = 0; sl < slices.size() && rc == LWB_OK; sl++) {
            // arena set sl & 1 of the slice's group was last read by the synthesis of slice sl - 2 or earlier, which
            // finished before that of slice sl - 1 was started
            const double e0 = now_s();
            rc = batch_entropy(b, sl & 1, jobs, slices[sl].data(), slices[sl].size(), plan, decoded, dec_status, &used);
            entropy_busy += now_s() - e0;
            if (synth.joinable()) synth.join();
            if (rc != LWB_OK || synth_rc != LWB_OK) break;
            const size_t g = used[0];
            BatchArena &ar = b->groups[g]->arena[sl & 1];
            in_bytes += ar.in_bytes;
            synth = std::thread([b, g, &ar, out_format, pcm, jobs, &plan, &decoded, &dec_status, &synth_rc, &synth_busy]() {
                const double s0 = now_s();
                const lwb_batch_io io = batch_io(b, g, ar, out_format, pcm);
                const int r = lwb_decode_chains(b->ctx, ar.chains.data(), ar.chains.size(), &io);
                synth_busy += now_s() - s0;
                if (r) { synth_rc = r; return; }
                job_results(jobs, ar, plan, decoded, dec_status);
            });
        }
        if (synth.joinable()) synth.join();
        b->t_entropy = entropy_busy;
        b->t_synth = synth_busy;
        b->in_bytes = in_bytes;
        if (rc) return rc;
        return synth_rc;
    });
}

// ---------------------------------------------------------------------------------------------
// debug taps for the known-answer tests of the reference's own unit tests (bitpacking.rs:316-334,
// :488-600, huffman_tree.rs:262-330, header.rs:650-671)
// ---------------------------------------------------------------------------------------------
// Timing aid (profiles/frontend_bench.py): decodes the n packets `reps` times inside one call, so that the number is the
// decoder's and not the caller's; vq != 0: records instead of dense residue vectors.  Returns seconds, < 0 on error.
extern "C" double lwf_debug_decode_loop(const lwf_headers *h, const uint8_t *const *packets, const size_t *lens, size_t n, int reps, int vq)
{
    if (!h || !packets || !lens) return -1.0;
    try {
        lwfb::PacketScratch s(h);
        size_t cap = 16;
        for (size_t i = 0; i < n; i++) cap = std::max(cap, lens[i] * 8 + 16);
        std::vector<lwb_vq_run> runs(cap);
        std::vector<uint16_t> ents(cap);
        const auto t0 = std::chrono::steady_clock::now();
        for (int r = 0; r < reps; r++)
            for (size_t i = 0; i < n; i++) {
                lwf_decoded_packet dp = s.packet();
                if (vq) dp.residue = nullptr;
                lwf::VqSink sink;
                sink.runs = runs.data(); sink.run_cap = cap; sink.entries = ents.data(); sink.ent_cap = cap;
                if (lwf::packet_decode(h->body(), packets[i], lens[i], &dp, vq ? &sink : nullptr)) return -2.0;
            }
        return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    } catch (...) {
        return -3.0;
    }
}

extern "C" float lwf_debug_float32_unpack(uint32_t v) { return lwf::float32_unpack(v); }
extern "C" uint32_t lwf_debug_lookup1_values(uint32_t entries, uint16_t dims) { return lwf::lookup1_values(entries, dims); }
extern "C" uint8_t lwf_debug_ilog(uint64_t v) { return lwf::ilog(v); }
// reads widths[i] bits each; returns how many reads succeeded
extern "C" size_t lwf_debug_read_bits(const uint8_t *data, size_t len, const uint8_t *widths, size_t n, uint64_t *out)
{
    lwf::BitReader rdr(data, len);
    size_t k = 0;
    for (; k < n; k++)
        if (!rdr.read(widths[k], &out[k])) break;
    return k;
}
// builds the tree from codeword lengths (returns the HuffmanError class, 0 = ok) and decodes symbols
// from `data` until it runs out
extern "C" int lwf_debug_huffman(const uint8_t *lengths, size_t n, const uint8_t *data, size_t len, uint32_t *out, size_t max_out,
                                 size_t *n_out)
{
    lwf::Huffman t;
    const int rc = t.load(std::vector<uint8_t>(lengths, lengths + n));
    if (n_out) *n_out = 0;
    if (rc || !data || !out || !n_out) return rc;
    lwf::BitReader rdr(data, len);
    while (*n_out < max_out) {
        uint32_t v;
        if (!t.read(rdr, &v)) break;
        out[(*n_out)++] = v;
    }
    return 0;
}
