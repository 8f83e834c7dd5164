// Baseline JPEG decoding on the GPU, byte-identical to PIL (libjpeg-turbo with PIL's defaults).
//
// The reference decodes every image on the CPU, Image.open(f).convert("RGB") (dirtorch/datasets/dataset.py:52,
// generic.py:246); at ~60 images/s per core that, not the network, limits extraction.  Here the host parses the
// markers (ITU-T T.81) and uploads the entropy-coded data of a whole batch in one copy; the kernels then
//   1. unstuff: drop the FF 00 stuffing, split at RSTn, check the restart numbering (one CTA per image);
//   2. Huffman-decode in parallel by self-synchronisation (Weissenberger & Schmidt, ICPP 2018): the bit stream of each
//      image is cut into subsequences of S bits; a thread decodes its subsequence from a guessed state (bit position,
//      block slot in the MCU, zig-zag index) and records the state at the next boundary; rounds then re-decode
//      subsequences whose predecessor's state changed, running on while their result differs from what is recorded,
//      until a round changes nothing: every recorded state is then the true one;
//   3. count the blocks of every subsequence, scan the counts, decode again writing de-zigzagged int16 coefficients;
//   4. turn DC differences into values by a scan per restart segment and component;
//   5. dequantise + ISLOW integer IDCT (libjpeg jidctint.c arithmetic, wrap-then-clamp range limit) into planes;
//   6. fancy upsampling (libjpeg jdsample.c) + YCbCr->RGB (jdcolor.c fixed-point tables) into uint8 HWC RGB.
// The arithmetic is restated in numpy by tests/jpeg_model.py, which equals PIL byte for byte.
//
// Segment ends.  A segment (restart interval) ends with fewer than 8 one-bits of padding; bits past its end read as
// ones here.  The host refuses tables holding an all-ones code (libjpeg's encoder never emits one), so at the padding
// no code matches, and a decoder moves to the next segment without knowing how many MCUs the segment holds.  Anywhere
// else, no matching code, a coefficient index past 63 or value bits beyond the end are errors: a decoder from a guessed
// state steps one bit and goes on (it resynchronises), the counting pass, which runs from exact states, flags the
// image, and so does a per-segment block count that differs from the header's.  libjpeg's repair of corrupt data
// (zero bits, skipped markers) is not reproduced: a flagged image is re-decoded by the caller with PIL.
#include <string.h>

#include <algorithm>
#include <vector>

#include "block.cuh"
#include "common.h"

namespace dirb {
namespace {

constexpr int FAST_BITS = 9;
constexpr int MAX_SLOTS = 6;           // blocks per MCU: 4 Y + Cb + Cr at most
constexpr int DEFAULT_SUBSEQ_BITS = 1024;
constexpr int ROUNDS_PER_CHECK = 4;

struct HuffTab {
  uint16_t fast[1 << FAST_BITS];       // (length << 8) | symbol for codes of at most FAST_BITS bits, 0 otherwise
  int32_t maxcode[18];                 // largest code of each length, -1 if none
  int32_t valoff[18];                  // symbol index = code + valoff[length]
  uint8_t vals[256];
};

struct ImgDesc {
  int64_t in_off;                      // entropy-coded bytes in the data region (also the unstuffed copy's offset)
  int64_t blk_off;                     // first coefficient block of the image
  int64_t plane_off[3];                // component planes (bytes)
  int64_t out_off;                     // RGB output (bytes, caller's buffer)
  int64_t sub_off;                     // first subsequence
  int32_t in_len, nsub, nblk;
  int32_t h, w, ncomp, bpm, mcux, mcuy, ri, nseg, seg_off, hmax, vmax, color;   // color 0 YCbCr, 1 RGB, 2 gray
  int32_t plane_w[3], comp_h[3], comp_w[3], hs[3], vs[3];
  int32_t slot_comp[MAX_SLOTS], slot_dy[MAX_SLOTS], slot_dx[MAX_SLOTS];
};

enum : int { ST_MARKER = 1, ST_RESTART = 2, ST_BLOCKS = 4, ST_CODE = 8 };

// ------------------------------------------------------------------------------------------------------ host parser

struct Comp {
  int id, hs, vs, tq, td, ta;
};

struct Parsed {
  int h = 0, w = 0, ncomp = 0, ri = 0, color = 0;
  Comp comp[3];
  int qt[4][64];
  bool qt_set[4] = {false, false, false, false};
  HuffTab dc[4], ac[4];
  bool dc_set[4] = {false, false, false, false}, ac_set[4] = {false, false, false, false};
  size_t scan_begin = 0, scan_end = 0;
};

const int kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                         41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                         30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
__constant__ int c_zigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                 41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// T.81 Annex C code assignment (libjpeg jpeg_make_d_derived_tbl) -> lookup tables.
int build_huff(const uint8_t* counts, const uint8_t* vals, int nvals, bool dc, HuffTab* t) {
  memset(t, 0, sizeof(*t));
  memcpy(t->vals, vals, nvals);
  int code = 0, k = 0;
  for (int len = 1; len <= 16; ++len) {
    const int n = counts[len - 1];
    t->maxcode[len] = -1;
    if (n) {
      t->valoff[len] = k - code;
      for (int i = 0; i < n; ++i, ++code, ++k) {
        DIRB_REQUIRE(code < (1 << len), DIRB200_EINVAL, "bad Huffman table");
        DIRB_REQUIRE(code != (1 << len) - 1, DIRB200_ENOTSUP, "Huffman table with an all-ones code");
        if (dc) DIRB_REQUIRE(vals[k] <= 15, DIRB200_EINVAL, "bad DC Huffman symbol");
        if (len <= FAST_BITS) {
          const int shift = FAST_BITS - len;
          for (int f = 0; f < (1 << shift); ++f) t->fast[(code << shift) | f] = static_cast<uint16_t>(len << 8 | vals[k]);
        }
      }
      t->maxcode[len] = code - 1;
    }
    code <<= 1;
  }
  t->maxcode[17] = 0x7fffffff;
  return 0;
}

int rd16(const uint8_t* p) { return (p[0] << 8) | p[1]; }

// Markers up to the first SOS.  Unsupported but well-formed inputs -> DIRB200_ENOTSUP; malformed -> DIRB200_EINVAL.
int parse_jpeg(const uint8_t* d, size_t n, Parsed* P) {
  DIRB_REQUIRE(d && n >= 4, DIRB200_EINVAL, "not a JPEG (too short)");
  DIRB_REQUIRE(d[0] == 0xFF && d[1] == 0xD8, DIRB200_EINVAL, "not a JPEG (no SOI)");
  size_t p = 2;
  bool jfif = false, sof = false;
  int adobe = -1;
  for (;;) {
    DIRB_REQUIRE(p + 2 <= n && d[p] == 0xFF, DIRB200_EINVAL, "bad or truncated marker at byte %zu", p);
    while (p + 2 <= n && d[p + 1] == 0xFF) ++p;                     // fill bytes
    DIRB_REQUIRE(p + 4 <= n, DIRB200_EINVAL, "truncated marker");
    const int m = d[p + 1];
    DIRB_REQUIRE(m != 0xD9 && m != 0x00 && !(m >= 0xD0 && m <= 0xD8) && m != 0x01, DIRB200_EINVAL,
                 "unexpected marker %02X before SOS", m);
    const size_t len = rd16(d + p + 2);
    DIRB_REQUIRE(len >= 2 && p + 2 + len <= n, DIRB200_EINVAL, "truncated segment (marker %02X)", m);
    const uint8_t* s = d + p + 4;
    const size_t sl = len - 2;
    if (m == 0xE0 && sl >= 14 && memcmp(s, "JFIF\0", 5) == 0) {   // libjpeg needs the whole 14-byte JFIF header
      jfif = true;
    } else if (m == 0xEE && sl >= 12 && memcmp(s, "Adobe", 5) == 0) {
      adobe = s[11];
    } else if (m == 0xDB) {                                         // DQT
      size_t q = 0;
      while (q < sl) {
        const int pq = s[q] >> 4, tq = s[q] & 15;
        DIRB_REQUIRE(pq <= 1 && tq <= 3 && q + 1 + (pq ? 128 : 64) <= sl, DIRB200_EINVAL, "bad DQT");
        for (int i = 0; i < 64; ++i)
          P->qt[tq][kZigzag[i]] = pq ? rd16(s + q + 1 + 2 * i) : s[q + 1 + i];
        P->qt_set[tq] = true;
        q += 1 + (pq ? 128 : 64);
      }
    } else if (m == 0xC4) {                                         // DHT
      size_t q = 0;
      while (q < sl) {
        DIRB_REQUIRE(q + 17 <= sl, DIRB200_EINVAL, "bad DHT");
        const int tc = s[q] >> 4, th = s[q] & 15;
        DIRB_REQUIRE(tc <= 1 && th <= 3, DIRB200_EINVAL, "bad DHT class/id");
        int nv = 0;
        for (int i = 0; i < 16; ++i) nv += s[q + 1 + i];
        DIRB_REQUIRE(nv <= 256 && q + 17 + nv <= sl, DIRB200_EINVAL, "bad DHT length");
        DIRB_TRY(build_huff(s + q + 1, s + q + 17, nv, tc == 0, tc ? &P->ac[th] : &P->dc[th]));
        (tc ? P->ac_set : P->dc_set)[th] = true;
        q += 17 + nv;
      }
    } else if (m == 0xDD) {                                         // DRI
      DIRB_REQUIRE(sl >= 2, DIRB200_EINVAL, "bad DRI");
      P->ri = rd16(s);
    } else if (m == 0xC0 || m == 0xC1) {                            // SOF0 / SOF1
      DIRB_REQUIRE(!sof && sl >= 6, DIRB200_EINVAL, "bad SOF");
      sof = true;
      DIRB_REQUIRE(s[0] == 8, DIRB200_ENOTSUP, "%d-bit samples", s[0]);
      P->h = rd16(s + 1);
      P->w = rd16(s + 3);
      P->ncomp = s[5];
      DIRB_REQUIRE(P->h > 0, DIRB200_ENOTSUP, "height defined by DNL");
      DIRB_REQUIRE(P->w > 0, DIRB200_EINVAL, "zero width");
      DIRB_REQUIRE(P->ncomp == 1 || P->ncomp == 3, DIRB200_ENOTSUP, "%d components", P->ncomp);
      DIRB_REQUIRE(sl >= 6 + 3 * static_cast<size_t>(P->ncomp), DIRB200_EINVAL, "bad SOF length");
      for (int c = 0; c < P->ncomp; ++c) {
        P->comp[c].id = s[6 + 3 * c];
        P->comp[c].hs = s[7 + 3 * c] >> 4;
        P->comp[c].vs = s[7 + 3 * c] & 15;
        P->comp[c].tq = s[8 + 3 * c];
        DIRB_REQUIRE(P->comp[c].hs >= 1 && P->comp[c].hs <= 4 && P->comp[c].vs >= 1 && P->comp[c].vs <= 4 &&
                     P->comp[c].tq <= 3, DIRB200_EINVAL, "bad component parameters");
      }
    } else if (m >= 0xC2 && m <= 0xCF && m != 0xC4 && m != 0xC8 && m != 0xCC) {
      return set_error("SOF%d (progressive, lossless, arithmetic or hierarchical) is not supported", m - 0xC0),
             DIRB200_ENOTSUP;
    } else if (m == 0xDA) {                                         // SOS
      DIRB_REQUIRE(sof, DIRB200_EINVAL, "SOS before SOF");
      DIRB_REQUIRE(sl >= 1 && sl >= 1 + 2 * static_cast<size_t>(s[0]) + 3, DIRB200_EINVAL, "bad SOS");
      const int ns = s[0];
      DIRB_REQUIRE(ns == P->ncomp, DIRB200_ENOTSUP, "multi-scan sequential JPEG");
      for (int i = 0; i < ns; ++i) {
        DIRB_REQUIRE(s[1 + 2 * i] == P->comp[i].id, DIRB200_ENOTSUP, "scan components out of frame order");
        P->comp[i].td = s[2 + 2 * i] >> 4;
        P->comp[i].ta = s[2 + 2 * i] & 15;
        DIRB_REQUIRE(P->comp[i].td <= 3 && P->comp[i].ta <= 3 && P->dc_set[P->comp[i].td] && P->ac_set[P->comp[i].ta] &&
                     P->qt_set[P->comp[i].tq], DIRB200_EINVAL, "scan refers to an undefined table");
      }
      const uint8_t* e = s + 1 + 2 * ns;
      DIRB_REQUIRE(e[0] == 0 && e[1] == 63 && e[2] == 0, DIRB200_ENOTSUP, "not a sequential DCT scan");
      if (P->ncomp == 3) {
        const Comp* c = P->comp;
        const bool chroma11 = c[1].hs == 1 && c[1].vs == 1 && c[2].hs == 1 && c[2].vs == 1;
        const bool luma = (c[0].hs == 1 && c[0].vs == 1) || (c[0].hs == 2 && c[0].vs == 1) || (c[0].hs == 2 && c[0].vs == 2);
        DIRB_REQUIRE(chroma11 && luma, DIRB200_ENOTSUP, "sampling %dx%d,%dx%d,%dx%d", c[0].hs, c[0].vs, c[1].hs,
                     c[1].vs, c[2].hs, c[2].vs);
        // libjpeg's colour-space rule for three components (jdapimin.c default_decompress_parms)
        if (jfif) P->color = 0;
        else if (adobe >= 0) P->color = adobe == 0 ? 1 : 0;
        else P->color = (c[0].id == 'R' && c[1].id == 'G' && c[2].id == 'B') ? 1 : 0;
      } else {
        P->color = 2;
      }
      P->scan_begin = p + 2 + len;
      // The entropy-coded data runs to the first marker other than RSTn (FF 00 is a stuffed data byte, FF FF a fill
      // byte).  That marker must be the EOI; whatever follows it (an MPF second image, a vendor trailer) is ignored,
      // as libjpeg ignores it.  A DNL or a further scan is left to PIL.
      size_t q = P->scan_begin;
      for (;;) {
        const void* ff = q < n ? memchr(d + q, 0xFF, n - q) : nullptr;
        DIRB_REQUIRE(ff, DIRB200_EINVAL, "truncated JPEG (no EOI after the scan)");
        const size_t f = static_cast<const uint8_t*>(ff) - d;
        size_t r = f;
        while (r + 1 < n && d[r + 1] == 0xFF) ++r;
        DIRB_REQUIRE(r + 1 < n, DIRB200_EINVAL, "truncated JPEG (no EOI after the scan)");
        const int mk = d[r + 1];
        if (mk == 0x00 || (mk >= 0xD0 && mk <= 0xD7)) {      // stuffing or RSTn: the unstuff kernel handles them
          q = r + 2;
          continue;
        }
        DIRB_REQUIRE(mk == 0xD9, DIRB200_ENOTSUP, "marker %02X after the scan (DNL or a further scan)", mk);
        P->scan_end = f;                                      // fill bytes before the EOI are not data
        return 0;
      }
    }
    p += 2 + len;
  }
}

// ---------------------------------------------------------------------------------------------------------- kernels

// 1. Unstuff: one CTA per image; tiles of 256 x 16 stuffed bytes.  segstart[seg_off + s] = first unstuffed byte of
// segment s, segstart[seg_off + nseg] = unstuffed length.
__global__ void __launch_bounds__(256) unstuff_kernel(const ImgDesc* __restrict__ imgs, const uint8_t* __restrict__ in,
                                                      uint8_t* __restrict__ out, int* __restrict__ segstart,
                                                      int* __restrict__ status) {
  __shared__ int warp_sums[256 / 32];
  const ImgDesc& im = imgs[blockIdx.x];
  if (im.nsub == 0) return;                                   // rejected by the host parser
  const uint8_t* src = in + im.in_off;
  uint8_t* dst = out + im.in_off;
  int* seg = segstart + im.seg_off;
  const int n = im.in_len;
  int kept_base = 0, rst_base = 0, bad = 0;
  for (int t0 = 0; t0 < n; t0 += 256 * 16) {
    const int p0 = t0 + threadIdx.x * 16;
    uint32_t keep = 0, rst = 0;                               // bit masks over the thread's 16 bytes
    for (int i = 0; i < 16; ++i) {
      const int p = p0 + i;
      if (p >= n) break;
      const int b = src[p], prev = p > 0 ? src[p - 1] : 0, next = p + 1 < n ? src[p + 1] : -1;
      if (b == 0xFF) {
        if (next == 0x00) keep |= 1u << i;
        else if (next >= 0xD0 && next <= 0xD7) rst |= 1u << i;
        else if (next != 0xFF) bad |= ST_MARKER;              // any other marker inside the scan, or a trailing FF
      } else if (prev == 0xFF && (b == 0x00 || (b >= 0xD0 && b <= 0xD7))) {
      } else {
        keep |= 1u << i;
      }
    }
    int tot_k, tot_r;
    const int nk = __popc(keep), nr = __popc(rst);
    const int kb = block_scan(nk, warp_sums, &tot_k) - nk;
    const int rb = block_scan(nr, warp_sums, &tot_r) - nr;
    int k = kept_base + kb, r = rst_base + rb;
    for (int i = 0; i < 16; ++i) {
      if (keep >> i & 1) dst[k++] = src[p0 + i];
      if (rst >> i & 1) {
        if (src[p0 + i + 1] != 0xD0 + (r & 7)) bad |= ST_RESTART;
        ++r;
        if (r < im.nseg) seg[r] = k;
        else bad |= ST_RESTART;
      }
    }
    kept_base += tot_k;
    rst_base += tot_r;
  }
  if (threadIdx.x == 0) {
    seg[0] = 0;
    seg[im.nseg] = kept_base;
    if (rst_base != im.nseg - 1) bad |= ST_RESTART;
  }
  if (bad) atomicOr(status + blockIdx.x, bad);
}

struct Dec {
  const ImgDesc* im;
  const uint8_t* data;                                        // unstuffed bytes of the image (4-byte aligned)
  const int* seg;                                             // segment starts (bytes), nseg + 1 entries
  const HuffTab* tabs;                                        // 3 DC + 3 AC
};

// 32 bits of the stream from bit `pos`; bits at or past `end` read as ones.
__device__ __forceinline__ uint32_t peek32(const uint8_t* data, uint32_t pos, uint32_t end) {
  const uint32_t* w = reinterpret_cast<const uint32_t*>(data);
  const uint32_t wi = pos >> 5;
  const uint64_t hi = __byte_perm(__ldg(w + wi), 0, 0x0123), lo = __byte_perm(__ldg(w + wi + 1), 0, 0x0123);
  uint32_t v = static_cast<uint32_t>(((hi << 32 | lo) << (pos & 31)) >> 32);
  if (pos + 32 > end) {
    const uint32_t valid = end > pos ? end - pos : 0;
    v |= valid >= 32 ? 0u : (0xffffffffu >> valid);
  }
  return v;
}

// Decodes one Huffman symbol from the top of v; returns (length << 8 | symbol) or 0 if no code matches.
__device__ __forceinline__ int huff_sym(const HuffTab* __restrict__ t, uint32_t v) {
  const int f = t->fast[v >> (32 - FAST_BITS)];
  if (f) return f;
  for (int len = FAST_BITS + 1; len <= 16; ++len) {
    const int code = static_cast<int>(v >> (32 - len));
    if (code <= t->maxcode[len]) return len << 8 | t->vals[code + t->valoff[len]];
  }
  return 0;
}

__device__ __forceinline__ uint64_t pack_state(uint32_t pos, int slot, int zz) {
  return static_cast<uint64_t>(pos) << 16 | static_cast<uint64_t>(slot) << 8 | static_cast<uint64_t>(zz);
}

enum Mode { M_SYNC = 0, M_COUNT = 1, M_WRITE = 2 };

// Decodes the codewords that start in bits [sub_begin, sub_end) of one image, from state `st`.  Returns the state at
// the first codeword start at or past sub_end.  M_COUNT adds completed blocks per segment into seg_cnt, returns their
// total in *nblocks and flags the image in *status when it meets an invalid code; M_WRITE writes coefficients of blocks
// blk0, blk0 + 1, ... (DC as a difference).
template <int MODE>
__device__ uint64_t decode_run(const Dec& D, uint64_t st, uint32_t sub_end, int* nblocks, int* seg_cnt, int16_t* coef,
                               int64_t blk0, int* status) {
  const ImgDesc& im = *D.im;
  uint32_t pos = static_cast<uint32_t>(st >> 16);
  int slot = static_cast<int>(st >> 8 & 0xff), zz = static_cast<int>(st & 0xff);
  const uint32_t total = static_cast<uint32_t>(D.seg[im.nseg]) * 8u;
  // segment holding pos: the last s with seg[s] * 8 <= pos
  int s = 0;
  {
    int lo = 0, hi = im.nseg - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (static_cast<uint32_t>(D.seg[mid]) * 8u <= pos) lo = mid; else hi = mid - 1;
    }
    s = lo;
  }
  uint32_t seg_end = static_cast<uint32_t>(D.seg[s + 1]) * 8u;
  int count = 0, seg_count = 0;
  int64_t blk = blk0;
  for (;;) {
    while (pos >= seg_end && s < im.nseg) {                  // next segment: the state is exact again
      if (MODE == M_COUNT && seg_count) atomicAdd(seg_cnt + s, seg_count);
      seg_count = 0;
      ++s;
      pos = s < im.nseg ? static_cast<uint32_t>(D.seg[s]) * 8u : total;
      seg_end = s < im.nseg ? static_cast<uint32_t>(D.seg[s + 1]) * 8u : total;
      slot = 0;
      zz = 0;
    }
    if (s >= im.nseg || pos >= sub_end) break;
    const uint32_t v = peek32(D.data, pos, seg_end);
    const int ci = im.slot_comp[slot];
    const int hs = huff_sym(D.tabs + (zz == 0 ? ci : 3 + ci), v);
    const int len = hs >> 8, sym = hs & 0xff;
    const int nbits = sym & 15;
    const int r = zz == 0 ? 0 : sym >> 4;
    if (!hs || pos + len + nbits > seg_end || (zz > 0 && nbits && zz + r > 63)) {
      if (v == 0xffffffffu && seg_end - pos < 8) {            // the one-bit padding: the segment ends here
        pos = seg_end;
        continue;
      }
      if (MODE == M_SYNC) {                                   // a guessed state: step one bit and resynchronise
        ++pos;
        continue;
      }
      if (MODE == M_COUNT) atomicOr(status, ST_CODE);         // the exact state meets corrupt data
      pos = seg_end;
      continue;
    }
    int val = 0;
    if (nbits) {
      const uint32_t raw = (v << len) >> (32 - nbits);
      val = raw < (1u << (nbits - 1)) ? static_cast<int>(raw) - (1 << nbits) + 1 : static_cast<int>(raw);
    }
    pos += len + nbits;
    if (zz == 0) {
      if (MODE == M_WRITE && blk < im.nblk) coef[blk * 64] = static_cast<int16_t>(val);
      zz = 1;
    } else if (nbits) {
      const int k = zz + r;
      if (MODE == M_WRITE && blk < im.nblk) coef[blk * 64 + c_zigzag[k]] = static_cast<int16_t>(val);
      zz = k + 1;
    } else {
      zz = r == 15 ? zz + 16 : 64;                            // ZRL / EOB
    }
    if (zz >= 64) {
      ++count;
      ++seg_count;
      ++blk;
      zz = 0;
      slot = slot + 1 == im.bpm ? 0 : slot + 1;
    }
  }
  if (MODE == M_COUNT && seg_count && s < im.nseg) atomicAdd(seg_cnt + s, seg_count);
  if (nblocks) *nblocks = count;
  return pack_state(pos, slot, zz);
}

struct SubCtx {
  const ImgDesc* imgs;
  int nimg;
  const uint8_t* data;
  const int* segstart;
  const HuffTab* tabs;
  int S;
};

// global subsequence index -> (image, local index); false for padding threads
__device__ __forceinline__ bool locate(const SubCtx& c, int64_t g, int* img, int* j) {
  int lo = 0, hi = c.nimg - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (c.imgs[mid].sub_off <= g) lo = mid; else hi = mid - 1;
  }
  const ImgDesc& im = c.imgs[lo];
  if (g < im.sub_off || g >= im.sub_off + im.nsub) return false;
  *img = lo;
  *j = static_cast<int>(g - im.sub_off);
  return true;
}

__device__ __forceinline__ Dec make_dec(const SubCtx& c, int img) {
  Dec d;
  d.im = c.imgs + img;
  d.data = c.data + d.im->in_off;
  d.seg = c.segstart + d.im->seg_off;
  d.tabs = c.tabs + static_cast<int64_t>(img) * 6;
  return d;
}

__device__ __forceinline__ uint64_t entry_state(const uint64_t* st, int64_t g, int j) {
  return j == 0 ? pack_state(0, 0, 0) : __ldcg(reinterpret_cast<const unsigned long long*>(st + g - 1));
}

// 2a. Every subsequence from a guessed state: its start bit, block slot 0, zig-zag index 0 (the exact state for the
// first subsequence of an image).  st[g] = state at the next subsequence's start.
__global__ void sync_init_kernel(SubCtx c, int64_t nsub_total, uint64_t* st, uint8_t* dirty, int* status) {
  const int64_t g = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  int img, j;
  if (g >= nsub_total || !locate(c, g, &img, &j) || status[img]) return;
  const Dec D = make_dec(c, img);
  const uint32_t b = static_cast<uint32_t>(j) * c.S;
  st[g] = decode_run<M_SYNC>(D, pack_state(b, 0, 0), b + c.S, nullptr, nullptr, nullptr, 0, nullptr);
  dirty[g] = 1;
}

// 2b. One synchronisation round.  A subsequence whose predecessor's state was written last round is decoded again
// from it; where the result differs from the recorded state, it is recorded and the thread runs on into the next
// subsequence, until its result equals the recorded one.  A round that writes nothing leaves every state exact.
__global__ void sync_round_kernel(SubCtx c, int64_t nsub_total, uint64_t* st, const uint8_t* dirty_in, uint8_t* dirty_out,
                                  int* writes, int round, const int* status) {
  if (round > 0 && __ldcg(writes + round - 1) == 0) return;
  const int64_t g = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  int img, j;
  if (g >= nsub_total || !locate(c, g, &img, &j) || j == 0 || status[img] || !dirty_in[g - 1]) return;
  const Dec D = make_dec(c, img);
  uint64_t in = entry_state(st, g, j);
  int n = 0;
  for (int k = j; k < D.im->nsub; ++k) {
    const uint64_t e = decode_run<M_SYNC>(D, in, static_cast<uint32_t>(k + 1) * c.S, nullptr, nullptr, nullptr, 0, nullptr);
    unsigned long long* slotp = reinterpret_cast<unsigned long long*>(st + D.im->sub_off + k);
    if (__ldcg(slotp) == e) break;
    __stcg(slotp, static_cast<unsigned long long>(e));
    dirty_out[D.im->sub_off + k] = 1;
    ++n;
    in = e;
  }
  if (n) atomicAdd(writes + round, n);
}

// 3a. Block count of every subsequence from its exact entry state; per-segment counts for the check.
__global__ void count_kernel(SubCtx c, int64_t nsub_total, const uint64_t* st, int* cnt, int* seg_cnt, int* status) {
  const int64_t g = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  int img, j;
  if (g >= nsub_total || !locate(c, g, &img, &j) || status[img]) return;
  const Dec D = make_dec(c, img);
  int n = 0;
  decode_run<M_COUNT>(D, entry_state(st, g, j), static_cast<uint32_t>(j + 1) * c.S, &n,
                      seg_cnt + D.im->seg_off, nullptr, 0, const_cast<int*>(status) + img);
  cnt[g] = n;
}

// 3b. One CTA per image: exclusive scan of the block counts (in place) and the per-segment block-count check.
__global__ void __launch_bounds__(256) scan_check_kernel(const ImgDesc* __restrict__ imgs, int* cnt,
                                                         const int* __restrict__ seg_cnt, int* status) {
  __shared__ int warp_sums[256 / 32];
  const ImgDesc& im = imgs[blockIdx.x];
  if (im.nsub == 0) return;
  int* c = cnt + im.sub_off;
  int base = 0;
  for (int t0 = 0; t0 < im.nsub; t0 += 256) {
    const int i = t0 + threadIdx.x;
    const int v = i < im.nsub ? c[i] : 0;
    int tot;
    const int e = block_scan(v, warp_sums, &tot) - v;
    if (i < im.nsub) c[i] = base + e;
    base += tot;
  }
  const int nmcu = im.mcux * im.mcuy;
  int bad = 0;
  for (int s = threadIdx.x; s < im.nseg; s += 256) {
    const int mcus = min(im.ri, nmcu - s * im.ri);
    if (seg_cnt[im.seg_off + s] != mcus * im.bpm) bad = ST_BLOCKS;
  }
  if (bad) atomicOr(status + blockIdx.x, bad);
}

// 3c. Decode again, writing coefficients.
__global__ void write_kernel(SubCtx c, int64_t nsub_total, const uint64_t* st, const int* blk_first, int16_t* coef,
                             const int* status) {
  const int64_t g = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  int img, j;
  if (g >= nsub_total || !locate(c, g, &img, &j) || status[img]) return;
  const Dec D = make_dec(c, img);
  decode_run<M_WRITE>(D, entry_state(st, g, j), static_cast<uint32_t>(j + 1) * c.S, nullptr, nullptr,
                      coef + D.im->blk_off * 64, blk_first[g], nullptr);
}

// 4. DC prediction: one warp per (image, restart segment); lane l takes MCU m0 + l of each 32-MCU tile and the warp
// scans each component's DC differences.
__global__ void dc_kernel(const ImgDesc* __restrict__ imgs, int nimg, const int* __restrict__ seg_base, int nseg_total,
                          int16_t* coef, const int* status) {
  const int wg = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (wg >= nseg_total) return;
  int lo = 0, hi = nimg - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (seg_base[mid] <= wg) lo = mid; else hi = mid - 1;
  }
  const ImgDesc& im = imgs[lo];
  const int s = wg - seg_base[lo];
  if (s >= im.nseg || status[lo]) return;
  const int nmcu = im.mcux * im.mcuy;
  const int m0 = s * im.ri, m1 = min(nmcu, m0 + im.ri);
  int16_t* cb = coef + im.blk_off * 64;
  int carry[3] = {0, 0, 0};
  for (int t = m0; t < m1; t += 32) {
    const int m = t + lane;
    int sum[3] = {0, 0, 0};
    if (m < m1)
      for (int b = 0; b < im.bpm; ++b) sum[im.slot_comp[b]] += cb[(static_cast<int64_t>(m) * im.bpm + b) * 64];
    for (int ci = 0; ci < im.ncomp; ++ci) {
      const int inc = warp_scan(sum[ci]);
      int run = carry[ci] + inc - sum[ci];
      if (m < m1)
        for (int b = 0; b < im.bpm; ++b)
          if (im.slot_comp[b] == ci) {
            int16_t* p = cb + (static_cast<int64_t>(m) * im.bpm + b) * 64;
            run += *p;
            *p = static_cast<int16_t>(run);
          }
      carry[ci] += __shfl_sync(0xffffffffu, inc, 31);
    }
  }
}

constexpr int F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299,
              F1847 = 15137, F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;

// One ISLOW 1-D pass (jidctint.c): x[0..7] in, o[0..7] out, descaled by `shift` with rounding.
__device__ __forceinline__ void idct8(const int* x, int* o, int shift) {
  int z2 = x[2], z3 = x[6];
  int z1 = (z2 + z3) * F0541;
  const int tmp2 = z1 - z3 * F1847, tmp3 = z1 + z2 * F0765;
  const int tmp0 = (x[0] + x[4]) * (1 << 13), tmp1 = (x[0] - x[4]) * (1 << 13);
  const int t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
  int a0 = x[7], a1 = x[5], a2 = x[3], a3 = x[1];
  z1 = a0 + a3;
  z2 = a1 + a2;
  z3 = a0 + a2;
  int z4 = a1 + a3;
  const int z5 = (z3 + z4) * F1175;
  a0 *= F0298;
  a1 *= F2053;
  a2 *= F3072;
  a3 *= F1501;
  z1 *= -F0899;
  z2 *= -F2562;
  z3 = z3 * -F1961 + z5;
  z4 = z4 * -F0390 + z5;
  a0 += z1 + z3;
  a1 += z2 + z4;
  a2 += z2 + z3;
  a3 += z1 + z4;
  const int r = 1 << (shift - 1);
  o[0] = (t10 + a3 + r) >> shift;
  o[7] = (t10 - a3 + r) >> shift;
  o[1] = (t11 + a2 + r) >> shift;
  o[6] = (t11 - a2 + r) >> shift;
  o[2] = (t12 + a1 + r) >> shift;
  o[5] = (t12 - a1 + r) >> shift;
  o[3] = (t13 + a0 + r) >> shift;
  o[4] = (t13 - a0 + r) >> shift;
}

// 5. Dequantise + IDCT: one thread per block; blockIdx.y = image.
__global__ void __launch_bounds__(128) idct_kernel(const ImgDesc* __restrict__ imgs, const int16_t* __restrict__ coef,
                                                   const int* __restrict__ qt, uint8_t* planes, const int* status) {
  const ImgDesc& im = imgs[blockIdx.y];
  if (status[blockIdx.y]) return;
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < im.nblk; b += gridDim.x * blockDim.x) {
    const int mcu = b / im.bpm, slot = b - mcu * im.bpm;
    const int ci = im.slot_comp[slot];
    const int my = mcu / im.mcux, mx = mcu - my * im.mcux;
    const int by = my * (im.ncomp == 1 ? 1 : im.vs[ci]) + im.slot_dy[slot];
    const int bx = mx * (im.ncomp == 1 ? 1 : im.hs[ci]) + im.slot_dx[slot];
    const int16_t* cp = coef + (im.blk_off + b) * 64;
    const int* q = qt + (static_cast<int64_t>(blockIdx.y) * 3 + ci) * 64;
    int ws[64];
    int4 raw[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) raw[i] = reinterpret_cast<const int4*>(cp)[i];
    const int16_t* cv = reinterpret_cast<const int16_t*>(raw);
#pragma unroll
    for (int col = 0; col < 8; ++col) {
      int x[8], o[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) x[k] = cv[k * 8 + col] * __ldg(q + k * 8 + col);
      idct8(x, o, 13 - 2);
#pragma unroll
      for (int k = 0; k < 8; ++k) ws[k * 8 + col] = o[k];
    }
    uint8_t* dst = planes + im.plane_off[ci] + static_cast<int64_t>(by) * 8 * im.plane_w[ci] + bx * 8;
#pragma unroll
    for (int row = 0; row < 8; ++row) {
      int o[8];
      idct8(ws + row * 8, o, 13 + 2 + 3);
      uint32_t lo = 0, hi = 0;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int w = ((o[k] + 512) & 1023) - 512;            // range limit: wrap to 10 bits, then clamp
        const uint32_t u = static_cast<uint32_t>(min(max(w + 128, 0), 255));
        if (k < 4) lo |= u << (8 * k); else hi |= u << (8 * (k - 4));
      }
      *reinterpret_cast<uint2*>(dst + static_cast<int64_t>(row) * im.plane_w[ci]) = make_uint2(lo, hi);
    }
  }
}

__device__ __forceinline__ int px(const uint8_t* p, int stride, int y, int x) { return p[static_cast<int64_t>(y) * stride + x]; }

// Fancy upsampling (jdsample.c) of a chroma sample at output (y, x); the component is fy x fx subsampled, ch x cw real
// samples.  Components at most 2 samples wide are replicated (libjpeg uses its plain upsampler there).
__device__ __forceinline__ int upsample_at(const uint8_t* p, int stride, int ch, int cw, int fy, int fx, int y, int x) {
  const int cy = y / fy, cx = x / fx;
  if (fx == 1 && fy == 1) return px(p, stride, cy, cx);
  if (cw <= 2) return px(p, stride, cy, cx);
  const int side = (x & 1) ? min(cx + 1, cw - 1) : max(cx - 1, 0);
  if (fy == 1) return (3 * px(p, stride, cy, cx) + px(p, stride, cy, side) + ((x & 1) ? 2 : 1)) >> 2;
  const int far = (y & 1) ? min(cy + 1, ch - 1) : max(cy - 1, 0);
  const int s_near = 3 * px(p, stride, cy, cx) + px(p, stride, far, cx);
  const int s_side = 3 * px(p, stride, cy, side) + px(p, stride, far, side);
  return (3 * s_near + s_side + ((x & 1) ? 7 : 8)) >> 4;
}

// 6. Upsample + colour conversion into the caller's HWC RGB buffer; blockIdx.y = image.
__global__ void color_kernel(const ImgDesc* __restrict__ imgs, const uint8_t* __restrict__ planes, uint8_t* out,
                             const int* status) {
  const ImgDesc& im = imgs[blockIdx.y];
  if (status[blockIdx.y]) return;
  const int64_t npx = static_cast<int64_t>(im.h) * im.w;
  uint8_t* o = out + im.out_off;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < npx;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int y = static_cast<int>(i / im.w), x = static_cast<int>(i - static_cast<int64_t>(y) * im.w);
    int r, g, b;
    const int c0 = px(planes + im.plane_off[0], im.plane_w[0], y, x);
    if (im.color == 2) {
      r = g = b = c0;
    } else {
      const int fy = im.vmax / im.vs[1], fx = im.hmax / im.hs[1];
      const int c1 = upsample_at(planes + im.plane_off[1], im.plane_w[1], im.comp_h[1], im.comp_w[1], fy, fx, y, x);
      const int c2 = upsample_at(planes + im.plane_off[2], im.plane_w[2], im.comp_h[2], im.comp_w[2], fy, fx, y, x);
      if (im.color == 1) {
        r = c0, g = c1, b = c2;
      } else {
        // jdcolor.c build_ycc_rgb_table: FIX(x) = round(x * 2^16), ONE_HALF = 2^15, arithmetic right shifts
        const int cb = c1 - 128, cr = c2 - 128;
        r = c0 + ((91881 * cr + 32768) >> 16);
        g = c0 + ((-22554 * cb + 32768 - 46802 * cr) >> 16);
        b = c0 + ((116130 * cb + 32768) >> 16);
      }
    }
    uint8_t* d = o + i * 3;
    d[0] = static_cast<uint8_t>(min(max(r, 0), 255));
    d[1] = static_cast<uint8_t>(min(max(g, 0), 255));
    d[2] = static_cast<uint8_t>(min(max(b, 0), 255));
  }
}

}  // namespace
}  // namespace dirb

using namespace dirb;

struct dirb200_jpeg_decoder {
  int device = 0;
  int subseq_bits = DEFAULT_SUBSEQ_BITS;
  uint8_t* stage = nullptr;                  // pinned staging of everything the batch uploads
  size_t stage_cap = 0;
  void* in_dev = nullptr;                    // device copy of the staging
  size_t in_cap = 0;
  void* ws_dev = nullptr;                    // device workspace
  size_t ws_cap = 0;
  cudaEvent_t staged = nullptr;              // the last upload has read the staging
  // layout of the last batch, for the debug export
  std::vector<ImgDesc> last;
  int16_t* coef_dev = nullptr;
};

namespace {

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

int fill_desc(const Parsed& P, ImgDesc* d) {
  memset(d, 0, sizeof(*d));
  d->h = P.h;
  d->w = P.w;
  d->ncomp = P.ncomp;
  d->color = P.color;
  if (P.ncomp == 1) {
    d->hmax = d->vmax = 1;
    d->hs[0] = d->vs[0] = 1;
    d->bpm = 1;
    d->slot_comp[0] = 0;
  } else {
    d->hmax = P.comp[0].hs;
    d->vmax = P.comp[0].vs;
    int k = 0;
    for (int c = 0; c < 3; ++c) {
      d->hs[c] = P.comp[c].hs;
      d->vs[c] = P.comp[c].vs;
      for (int yy = 0; yy < d->vs[c]; ++yy)
        for (int xx = 0; xx < d->hs[c]; ++xx, ++k) {
          d->slot_comp[k] = c;
          d->slot_dy[k] = yy;
          d->slot_dx[k] = xx;
        }
    }
    d->bpm = k;
  }
  d->mcux = static_cast<int>(ceil_div(P.w, 8 * d->hmax));
  d->mcuy = static_cast<int>(ceil_div(P.h, 8 * d->vmax));
  const int nmcu = d->mcux * d->mcuy;
  d->ri = P.ri > 0 ? std::min(P.ri, nmcu) : nmcu;
  d->nseg = static_cast<int>(ceil_div(nmcu, d->ri));
  d->nblk = nmcu * d->bpm;
  for (int c = 0; c < P.ncomp; ++c) {
    d->plane_w[c] = d->mcux * d->hs[c] * 8;
    d->comp_h[c] = static_cast<int>(ceil_div(static_cast<int64_t>(P.h) * d->vs[c], d->vmax));
    d->comp_w[c] = static_cast<int>(ceil_div(static_cast<int64_t>(P.w) * d->hs[c], d->hmax));
  }
  return 0;
}

}  // namespace

extern "C" {

int dirb200_jpeg_probe(const uint8_t* data, size_t size, int info[8]) {
  DIRB_REQUIRE(info, DIRB200_EINVAL, "info is NULL");
  memset(info, 0, 8 * sizeof(int));
  Parsed* P = new Parsed;
  const int s = parse_jpeg(data, size, P);
  info[0] = P->h;
  info[1] = P->w;
  info[2] = P->ncomp;
  info[3] = P->ncomp ? P->comp[0].hs : 0;
  info[4] = P->ncomp ? P->comp[0].vs : 0;
  info[5] = P->ri;
  info[6] = P->color;
  info[7] = s == 0 ? static_cast<int>(P->scan_end - P->scan_begin) : 0;
  delete P;
  return s;
}

int dirb200_jpeg_decoder_create(int device, dirb200_jpeg_decoder** out) {
  DIRB_REQUIRE(out, DIRB200_EINVAL, "out is NULL");
  *out = nullptr;
  DIRB_TRY(dirb200_device_check(device));
  DIRB_CUDA(cudaSetDevice(device));
  auto* d = new dirb200_jpeg_decoder;
  d->device = device;
  if (cudaEventCreateWithFlags(&d->staged, cudaEventDisableTiming) != cudaSuccess) {
    delete d;
    DIRB_REQUIRE(false, cudaErrorMemoryAllocation, "cudaEventCreate failed");
  }
  *out = d;
  return 0;
}

int dirb200_jpeg_decoder_set_option(dirb200_jpeg_decoder* d, const char* key, double value) {
  DIRB_REQUIRE(d && key, DIRB200_EINVAL, "bad arguments");
  if (!strcmp(key, "subseq_bits")) {
    DIRB_REQUIRE(value >= 64 && value <= (1 << 20) && static_cast<int>(value) % 32 == 0, DIRB200_EINVAL,
                 "subseq_bits must be a multiple of 32 in [64, 2^20]");
    d->subseq_bits = static_cast<int>(value);
  } else {
    DIRB_REQUIRE(false, DIRB200_EKEY, "unknown jpeg decoder option '%s'", key);
  }
  return 0;
}

int dirb200_jpeg_decoder_decode(dirb200_jpeg_decoder* d, int n, const uint8_t* const* data_host, const size_t* sizes_host,
                        uint8_t* out_dev, const int64_t* out_offsets_host, int* status_dev, int* rounds_out,
                        void* stream_) {
  DIRB_REQUIRE(d && n > 0 && data_host && sizes_host && out_dev && out_offsets_host && status_dev, DIRB200_EINVAL,
               "bad arguments");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DIRB_CUDA(cudaSetDevice(d->device));
  const int S = d->subseq_bits;
  // host: parse every image; lay out the upload and the workspace
  std::vector<ImgDesc> descs(n);
  std::vector<int> status(n, 0);
  std::vector<Parsed> parsed(n);
  size_t data_bytes = 0;
  int64_t nsub = 0, nblk = 0, planes = 0;
  int nseg = 0, nseg_pts = 0;
  std::vector<int> seg_base(n + 1, 0);
  for (int i = 0; i < n; ++i) {
    ImgDesc& D = descs[i];
    const int s = parse_jpeg(data_host[i], sizes_host[i], &parsed[i]);
    if (s != 0) {
      // an empty entry at the running offsets: locate() and dc_kernel binary-search non-decreasing offsets for the
      // last entry at or below an index, so an entry with no subsequences, blocks or segments is never found
      memset(&D, 0, sizeof(D));
      D.in_off = static_cast<int64_t>(data_bytes);
      D.sub_off = nsub;
      D.blk_off = nblk;
      D.seg_off = nseg_pts;
      status[i] = s;
      seg_base[i + 1] = nseg;
      continue;
    }
    fill_desc(parsed[i], &D);
    D.in_off = static_cast<int64_t>(data_bytes);
    D.in_len = static_cast<int>(parsed[i].scan_end - parsed[i].scan_begin);
    data_bytes += align_up(static_cast<size_t>(D.in_len) + 16, 16);
    D.sub_off = nsub;
    D.nsub = static_cast<int>(std::max<int64_t>(1, ceil_div(static_cast<int64_t>(D.in_len) * 8, S)));
    nsub += D.nsub;
    D.blk_off = nblk;
    nblk += D.nblk;
    for (int c = 0; c < D.ncomp; ++c) {
      D.plane_off[c] = planes;
      planes += static_cast<int64_t>(D.plane_w[c]) * D.mcuy * D.vs[c] * 8;
    }
    D.out_off = out_offsets_host[i];
    D.seg_off = nseg_pts;
    nseg_pts += D.nseg + 1;
    nseg += D.nseg;
    seg_base[i + 1] = nseg;
  }
  // upload: descs | tables | quant | seg_base | status | data
  const size_t o_desc = 0;
  const size_t o_tab = align_up(o_desc + sizeof(ImgDesc) * n, 16);
  const size_t o_qt = align_up(o_tab + sizeof(HuffTab) * 6 * n, 16);
  const size_t o_segb = align_up(o_qt + sizeof(int) * 64 * 3 * n, 16);
  const size_t o_stat = align_up(o_segb + sizeof(int) * (n + 1), 16);
  const size_t o_data = align_up(o_stat + sizeof(int) * n, 16);
  const size_t up_bytes = o_data + data_bytes;
  if (up_bytes > d->stage_cap) {
    DIRB_CUDA(cudaEventSynchronize(d->staged));
    if (d->stage) DIRB_CUDA(cudaFreeHost(d->stage));
    d->stage = nullptr;
    d->stage_cap = 0;
    DIRB_CUDA(cudaMallocHost(reinterpret_cast<void**>(&d->stage), up_bytes * 2));
    d->stage_cap = up_bytes * 2;
  } else {
    DIRB_CUDA(cudaEventSynchronize(d->staged));             // the previous upload has left the staging
  }
  uint8_t* st = d->stage;
  memcpy(st + o_desc, descs.data(), sizeof(ImgDesc) * n);
  HuffTab* tabs = reinterpret_cast<HuffTab*>(st + o_tab);
  int* qts = reinterpret_cast<int*>(st + o_qt);
  for (int i = 0; i < n; ++i) {
    if (status[i]) continue;
    const Parsed& P = parsed[i];
    for (int c = 0; c < P.ncomp; ++c) {
      tabs[i * 6 + c] = P.dc[P.comp[c].td];
      tabs[i * 6 + 3 + c] = P.ac[P.comp[c].ta];
      memcpy(qts + (i * 3 + c) * 64, P.qt[P.comp[c].tq], 64 * sizeof(int));
    }
    uint8_t* dst = st + o_data + descs[i].in_off;
    memcpy(dst, data_host[i] + P.scan_begin, descs[i].in_len);
    memset(dst + descs[i].in_len, 0, align_up(static_cast<size_t>(descs[i].in_len) + 16, 16) - descs[i].in_len);
  }
  memcpy(st + o_segb, seg_base.data(), sizeof(int) * (n + 1));
  memcpy(st + o_stat, status.data(), sizeof(int) * n);
  DIRB_TRY(grow_device(&d->in_dev, &d->in_cap, up_bytes));
  uint8_t* in = static_cast<uint8_t*>(d->in_dev);
  DIRB_CUDA(cudaMemcpyAsync(in, st, up_bytes, cudaMemcpyHostToDevice, stream));
  DIRB_CUDA(cudaEventRecord(d->staged, stream));
  DIRB_CUDA(cudaMemcpyAsync(status_dev, st + o_stat, sizeof(int) * n, cudaMemcpyHostToDevice, stream));
  // workspace: unstuffed data | segstart | seg_cnt | states | counts | dirty x2 | writes | coef | planes
  const int max_rounds = 1 << 16;
  const size_t w_un = 0;
  const size_t w_seg = align_up(w_un + data_bytes, 16);
  const size_t w_segc = align_up(w_seg + sizeof(int) * std::max(nseg_pts, 1), 16);
  const size_t w_st = align_up(w_segc + sizeof(int) * std::max(nseg_pts, 1), 16);   // indexed like segstart
  const size_t w_cnt = align_up(w_st + sizeof(uint64_t) * std::max<int64_t>(nsub, 1), 16);
  const size_t w_d0 = align_up(w_cnt + sizeof(int) * std::max<int64_t>(nsub, 1), 16);
  const size_t w_d1 = align_up(w_d0 + std::max<int64_t>(nsub, 1), 16);
  const size_t w_wr = align_up(w_d1 + std::max<int64_t>(nsub, 1), 16);
  const size_t w_coef = align_up(w_wr + sizeof(int) * max_rounds, 16);
  const size_t w_pl = align_up(w_coef + sizeof(int16_t) * 64 * std::max<int64_t>(nblk, 1), 16);
  const size_t ws_bytes = w_pl + std::max<int64_t>(planes, 1);
  DIRB_TRY(grow_device(&d->ws_dev, &d->ws_cap, ws_bytes));
  uint8_t* ws = static_cast<uint8_t*>(d->ws_dev);
  const ImgDesc* g_desc = reinterpret_cast<const ImgDesc*>(in + o_desc);
  SubCtx c;
  c.imgs = g_desc;
  c.nimg = n;
  c.data = ws + w_un;
  c.segstart = reinterpret_cast<const int*>(ws + w_seg);
  c.tabs = reinterpret_cast<const HuffTab*>(in + o_tab);
  c.S = S;
  int* segc = reinterpret_cast<int*>(ws + w_segc);
  uint64_t* states = reinterpret_cast<uint64_t*>(ws + w_st);
  int* cnt = reinterpret_cast<int*>(ws + w_cnt);
  uint8_t* dirty[2] = {ws + w_d0, ws + w_d1};
  int* writes = reinterpret_cast<int*>(ws + w_wr);
  int16_t* coef = reinterpret_cast<int16_t*>(ws + w_coef);
  uint8_t* pl = ws + w_pl;

  DIRB_CUDA(cudaMemsetAsync(ws + w_un, 0xFF, data_bytes, stream));     // padding past each stream reads as ones
  DIRB_CUDA(cudaMemsetAsync(segc, 0, sizeof(int) * std::max(nseg_pts, 1), stream));
  DIRB_CUDA(cudaMemsetAsync(coef, 0, sizeof(int16_t) * 64 * std::max<int64_t>(nblk, 1), stream));
  unstuff_kernel<<<n, 256, 0, stream>>>(g_desc, in + o_data, ws + w_un, reinterpret_cast<int*>(ws + w_seg), status_dev);
  const unsigned gsub = static_cast<unsigned>(ceil_div(std::max<int64_t>(nsub, 1), 128));
  sync_init_kernel<<<gsub, 128, 0, stream>>>(c, nsub, states, dirty[0], status_dev);
  count_launch(2);
  // Rounds go out in groups; one host wait per group reads how many states each round changed.  The rounds of a group
  // after the first one that changed nothing return at once.
  int rounds = 0, changing = 0;
  std::vector<int> wr(ROUNDS_PER_CHECK);
  for (;;) {
    const int r0 = rounds;
    for (int k = 0; k < ROUNDS_PER_CHECK; ++k, ++rounds) {
      DIRB_CUDA(cudaMemsetAsync(dirty[(rounds + 1) & 1], 0, std::max<int64_t>(nsub, 1), stream));
      DIRB_CUDA(cudaMemsetAsync(writes + rounds, 0, sizeof(int), stream));
      sync_round_kernel<<<gsub, 128, 0, stream>>>(c, nsub, states, dirty[rounds & 1], dirty[(rounds + 1) & 1], writes,
                                                  rounds, status_dev);
      count_launch();
    }
    DIRB_CUDA(cudaMemcpyAsync(wr.data(), writes + r0, sizeof(int) * ROUNDS_PER_CHECK, cudaMemcpyDeviceToHost, stream));
    DIRB_CUDA(cudaStreamSynchronize(stream));
    for (int k = 0; k < ROUNDS_PER_CHECK; ++k)
      if (wr[k]) changing = r0 + k + 1;
    if (wr[ROUNDS_PER_CHECK - 1] == 0) break;
    DIRB_REQUIRE(rounds + ROUNDS_PER_CHECK <= max_rounds, DIRB200_EOVERFLOW, "Huffman synchronisation did not converge");
  }
  if (rounds_out) *rounds_out = changing;
  count_kernel<<<gsub, 128, 0, stream>>>(c, nsub, states, cnt, segc, status_dev);
  scan_check_kernel<<<n, 256, 0, stream>>>(g_desc, cnt, segc, status_dev);
  write_kernel<<<gsub, 128, 0, stream>>>(c, nsub, states, cnt, coef, status_dev);
  const int* segb = reinterpret_cast<const int*>(in + o_segb);
  dc_kernel<<<static_cast<unsigned>(ceil_div(std::max(nseg, 1), 4)), 128, 0, stream>>>(g_desc, n, segb, nseg, coef,
                                                                                         status_dev);
  int max_blk = 1;
  int64_t max_px = 1;
  for (const ImgDesc& D : descs) {
    max_blk = std::max(max_blk, D.nblk);
    max_px = std::max<int64_t>(max_px, static_cast<int64_t>(D.h) * D.w);
  }
  idct_kernel<<<dim3(static_cast<unsigned>(std::min<int64_t>(ceil_div(max_blk, 128), 1024)), n), 128, 0, stream>>>(
      g_desc, coef, reinterpret_cast<const int*>(in + o_qt), pl, status_dev);
  color_kernel<<<dim3(static_cast<unsigned>(std::min<int64_t>(ceil_div(max_px, 256), 2048)), n), 256, 0, stream>>>(
      g_desc, pl, out_dev, status_dev);
  count_launch(6);
  DIRB_CUDA(cudaGetLastError());
  d->last = descs;
  d->coef_dev = coef;
  return 0;
}

int dirb200_jpeg_debug_coefficients(dirb200_jpeg_decoder* d, int image, int16_t* dst_dev, size_t capacity, int* nblocks,
                                    void* stream) {
  DIRB_REQUIRE(d && nblocks && image >= 0 && image < static_cast<int>(d->last.size()), DIRB200_EINVAL, "bad arguments");
  const ImgDesc& D = d->last[image];
  *nblocks = D.nblk;
  if (!dst_dev) return 0;
  const size_t bytes = sizeof(int16_t) * 64 * static_cast<size_t>(D.nblk);
  DIRB_REQUIRE(capacity >= bytes, DIRB200_EINVAL, "capacity %zu < %zu bytes", capacity, bytes);
  DIRB_CUDA(cudaMemcpyAsync(dst_dev, d->coef_dev + D.blk_off * 64, bytes, cudaMemcpyDeviceToDevice,
                            static_cast<cudaStream_t>(stream)));
  return 0;
}

int dirb200_jpeg_decoder_destroy(dirb200_jpeg_decoder* d) {
  if (!d) return 0;
  cudaSetDevice(d->device);
  if (d->staged) {
    cudaEventSynchronize(d->staged);
    cudaEventDestroy(d->staged);
  }
  if (d->stage) cudaFreeHost(d->stage);
  if (d->in_dev) cudaFree(d->in_dev);
  if (d->ws_dev) cudaFree(d->ws_dev);
  delete d;
  return 0;
}

}  // extern "C"
