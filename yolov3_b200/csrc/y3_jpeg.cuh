// yolov3_b200 — baseline JPEG decode, the parts shared by the device kernels (csrc/y3_jpeg.cu) and a plain C++ build
// (tests/test_jpeg_cpu.py compiles this header with g++ and runs every kernel's per-thread step on the host against cv2).
//
// What is restated bit for bit from libjpeg-turbo 3.x with its defaults (the decoder behind cv2.imread / cv2.imdecode):
//  * Huffman decode (jdhuff.c): canonical codes, HUFF_EXTEND, DC differences summed per component in MCU order and reset at
//    each restart, the sum kept as a wrapping int and stored as a 16-bit JCOEF;
//  * jpeg_idct_islow (jidctint.c): 13-bit constants, PASS1_BITS = 2, all-zero column / row short cuts, 64-bit products, the
//    +128 level shift and range limit through the 1024-entry table indexed by (x & 1023);
//  * fancy upsampling (jdsample.c): h2v1 and h2v2 triangle filters with the alternating biases when the chroma row is wider
//    than 2 samples (box replication otherwise), h1v2 triangle, 4x1 box; edges replicated at the component's real size;
//  * YCbCr -> RGB (jdcolor.c): the 16-fraction-bit tables, rounded;
//  * cv2's EXIF orientation remap (flip / transpose).
#pragma once
#include <stdint.h>
#include <string.h>

#include "../../include/yolov3_b200.h"

#ifdef __CUDACC__
#define Y3J_HD __host__ __device__ __forceinline__
#else
#define Y3J_HD inline
#endif

namespace y3 {
namespace jpeg {

constexpr int kSubBits = 512;  // bits per Huffman subsequence (one thread each)

struct Huff {                  // one Huffman table, as the device reads it
  uint16_t lut[512];           // 9-bit lookahead: (code length << 8) | symbol, 0 for longer codes
  int32_t maxcode[18];         // largest code of each length, -1 if none; [17] sentinel
  int32_t valoff[18];          // symbol index - code, per length
  uint8_t vals[256];
};
struct Tables {
  uint16_t quant[3][64];       // per component, natural order
  Huff huff[4];                // DC 0, DC 1, AC 0, AC 1
};
static_assert(sizeof(Tables) == Y3_JPEG_TABLE_BYTES, "table blob size");

// natural index of each zig-zag index, by walking the diagonals
Y3J_HD void zigzag_table(uint8_t* nat) {
  int r = 0, c = 0;
  for (int z = 0; z < 64; ++z) {
    nat[z] = static_cast<uint8_t>(r * 8 + c);
    if (((r + c) & 1) == 0) {
      if (c == 7) ++r;
      else if (r == 0) ++c;
      else { --r; ++c; }
    } else {
      if (r == 7) ++c;
      else if (c == 0) ++r;
      else { ++r; --c; }
    }
  }
}

// ---------------------------------------------------------------------------------------------------- workspace layout
struct Layout {
  int64_t unst, segsub, entry, exitv, count, flags, coef, plane[3], total;
  int32_t n_sub_max, pitch[3], rows[3];
};
Y3J_HD int64_t up256(int64_t v) { return (v + 255) & ~int64_t(255); }
Y3J_HD Layout layout(const y3_jpeg_geom& g) {
  Layout L;
  L.n_sub_max = static_cast<int32_t>(static_cast<int64_t>(g.unstuffed_len) * 8 / kSubBits) + g.n_segs + 1;
  int64_t o = 0;
  L.unst = o;   o += up256(g.unstuffed_len + 8);
  L.segsub = o; o += up256(4 * (static_cast<int64_t>(g.n_segs) + 1));
  L.entry = o;  o += up256(8 * static_cast<int64_t>(L.n_sub_max));
  L.exitv = o;  o += up256(8 * static_cast<int64_t>(L.n_sub_max));
  L.count = o;  o += up256(4 * static_cast<int64_t>(L.n_sub_max));
  L.flags = o;  o += up256(4 * static_cast<int64_t>(L.n_sub_max));
  L.coef = o;   o += up256(128 * static_cast<int64_t>(g.n_blocks));
  for (int c = 0; c < 3; ++c) {
    const int h = c == 0 ? g.hmax : 1, v = c == 0 ? g.vmax : 1;
    L.pitch[c] = g.mcus_x * h * 8;
    L.rows[c] = g.mcus_y * v * 8;
    L.plane[c] = o;
    if (c < g.ncomp) o += up256(static_cast<int64_t>(L.pitch[c]) * L.rows[c]);
  }
  L.total = o;
  return L;
}

// block b of an MCU -> component, and the block's (x, y) inside the MCU
Y3J_HD int mcu_comp(const y3_jpeg_geom& g, int b) { return b < g.hmax * g.vmax ? 0 : b - g.hmax * g.vmax + 1; }

// ------------------------------------------------------------------------------------------------------ unstuffing
// byte i of the entropy-coded data survives unless it is the 0x00 after a 0xFF, a 0xFF that starts a marker or fills,
// or the code byte of an RSTn marker
Y3J_HD bool keep_byte(const uint8_t* d, int i, int n) {
  const int c = d[i];
  const int prev = i > 0 ? d[i - 1] : 0;
  if (prev == 0xFF && (c == 0x00 || (c >= 0xD0 && c <= 0xD7))) return false;
  if (c == 0xFF && (i + 1 >= n || d[i + 1] != 0x00)) return false;
  return true;
}

// ---------------------------------------------------------------------------------------------------- Huffman decode
// decoder state between symbols: bit position in the segment, block of the MCU, zig-zag index
Y3J_HD uint64_t pack_state(int p, int b, int z) {
  return static_cast<uint64_t>(static_cast<uint32_t>(p)) << 16 | static_cast<uint64_t>(b) << 8 | static_cast<uint64_t>(z);
}
Y3J_HD int st_p(uint64_t s) { return static_cast<int>(s >> 16); }
Y3J_HD int st_b(uint64_t s) { return static_cast<int>((s >> 8) & 0xFF); }
Y3J_HD int st_z(uint64_t s) { return static_cast<int>(s & 0xFF); }

// 32 bits starting at bit p of a segment of nbytes bytes, zeros past its end (as libjpeg pads)
Y3J_HD uint32_t peek32(const uint8_t* seg, int nbytes, int p) {
  const int i = p >> 3;
  uint64_t v = 0;
#pragma unroll
  for (int k = 0; k < 5; ++k) v = v << 8 | (i + k < nbytes ? seg[i + k] : 0u);
  return static_cast<uint32_t>(v >> (8 - (p & 7)));
}

Y3J_HD int extend(uint32_t v, int s) {  // HUFF_EXTEND
  return s == 0 ? 0 : (v < (1u << (s - 1)) ? static_cast<int>(v) - (1 << s) + 1 : static_cast<int>(v));
}

// decodes one symbol at the top of w: returns (length << 8 | symbol), or 0 for an invalid code
Y3J_HD int huff_decode(const Huff& h, uint32_t w) {
  const int e = h.lut[w >> 23];
  if (e) return e;
  int l = 10;
  int32_t code = static_cast<int32_t>(w >> 22);
  while (l <= 16 && code > h.maxcode[l]) code = static_cast<int32_t>(w >> (32 - ++l));
  if (l > 16) return 0;
  return l << 8 | h.vals[(code + h.valoff[l]) & 0xFF];
}

struct SubResult {
  uint64_t exit;
  int32_t blocks;  // blocks completed
  int32_t err;
};

// canon[b]: the smallest block of the MCU from which every later block uses the same Huffman tables as from b (the table sequence
// repeats with the MCU, so comparing one MCU's worth suffices): decoding from either parses the bits identically, and the
// blocks land by their count, not by b.  Exit states carry canon[b].  So where components share their tables, a
// subsequence that started at the wrong block of the MCU still reaches the sequential decode's state, and the rounds need
// not carry the right b along the whole segment, one subsequence per round.
// canon[b] for one block of the MCU (at most 6): the MCU's table pairs packed 2 bits per block, rotations compared
Y3J_HD int canonical_block(const y3_jpeg_geom& g, int b) {
  const int n = g.blocks_per_mcu;
  uint32_t seq = 0;
  for (int k = 0; k < n; ++k) {
    const int c = mcu_comp(g, k);
    seq |= static_cast<uint32_t>(g.comp_dc[c] | g.comp_ac[c] << 1) << (2 * k);
  }
  const uint32_t mask = (1u << (2 * n)) - 1u;
  const auto rot = [&](int r) { return r == 0 ? seq : ((seq >> (2 * r)) | (seq << (2 * (n - r)))) & mask; };
  const uint32_t want = rot(b);
  int c = 0;
  while (rot(c) != want) ++c;
  return c;
}

// Decodes one subsequence from `entry` until the position reaches `end` (not the segment's last subsequence) or the
// segment ends (its last: an MCU boundary followed by at most 7 one-bits).  kWrite: store every zig-zag index the
// subsequence passes — the coefficient or 0 — into the blocks from `blk0` on (the DC difference at index 0).
template <bool kWrite>
Y3J_HD SubResult decode_sub(const y3_jpeg_geom& g, const Tables& T, const uint8_t* nat, const uint8_t* canon,
                            const uint8_t* seg, int nbytes, int end, bool last, uint64_t entry, int16_t* coef, int blk0) {
  const int nbits = nbytes * 8;
  int p = st_p(entry), b = st_b(entry), z = st_z(entry);
  SubResult r{0, 0, 0};
  int blk = blk0;
  for (;;) {
    if (!last && p >= end) break;
    if (b == 0 && z == 0) {
      const int rem = nbits - p;
      if (rem <= 7 && (rem <= 0 || (peek32(seg, nbytes, p) >> (32 - rem)) == (1u << rem) - 1u)) {
        if (rem < 0) r.err = 1;
        p = nbits;
        break;
      }
    }
    const int c = mcu_comp(g, b);
    const uint32_t w = peek32(seg, nbytes, p);
    int16_t* blkc = coef + static_cast<int64_t>(blk) * 64;
    const bool wr = kWrite && blk < g.n_blocks;
    if (z == 0) {
      const int e = huff_decode(T.huff[g.comp_dc[c]], w);
      if (!e) { r.err = 1; break; }
      const int len = e >> 8, s = e & 15;
      const uint32_t v = s ? (w << len) >> (32 - s) : 0u;
      if (wr) blkc[0] = static_cast<int16_t>(extend(v, s));
      p += len + s;
      z = 1;
    } else {
      const int e = huff_decode(T.huff[2 + g.comp_ac[c]], w);
      if (!e) { r.err = 1; break; }
      const int len = e >> 8, rs = e & 0xFF, run = rs >> 4, s = rs & 15;
      int nz = s ? z + run : (run == 15 ? z + 16 : 64);
      if (nz > (s ? 63 : 64)) { r.err = 1; break; }
      if (wr)
        for (int k = z; k < nz; ++k) blkc[nat[k]] = 0;
      if (s) {
        const uint32_t v = (w << len) >> (32 - s);
        if (wr) blkc[nat[nz]] = static_cast<int16_t>(extend(v, s));
        ++nz;
      }
      p += len + s;
      z = nz;
    }
    if (p > nbits) { r.err = 1; break; }
    if (z >= 64) {
      z = 0;
      b = b + 1 == g.blocks_per_mcu ? 0 : b + 1;
      ++r.blocks;
      ++blk;
    }
  }
  r.exit = r.err ? pack_state(end, 0, 0) : pack_state(p, canon[b], z);
  return r;
}

// ------------------------------------------------------------------------------------------------------------ IDCT
// jpeg_idct_islow.  Pass 1: column `col` of the dequantised block into ws (int, natural order); pass 2: row `row` of ws
// into 8 output samples.
constexpr int64_t F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299,
                  F1847 = 15137, F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;

Y3J_HD int range_limit(int64_t x) {  // libjpeg's IDCT range-limit table, indexed by (x & 1023) with +128 folded in
  const int i = static_cast<int>(x & 1023);
  return i < 128 ? i + 128 : (i < 512 ? 255 : (i < 896 ? 0 : i - 896));
}

Y3J_HD void idct_col(const int16_t* blk, const uint16_t* q, int col, int* ws) {
  int64_t in[8];
#pragma unroll
  for (int r = 0; r < 8; ++r) in[r] = static_cast<int64_t>(blk[r * 8 + col]) * static_cast<int64_t>(q[r * 8 + col]);
  if (blk[8 + col] == 0 && blk[16 + col] == 0 && blk[24 + col] == 0 && blk[32 + col] == 0 && blk[40 + col] == 0 &&
      blk[48 + col] == 0 && blk[56 + col] == 0) {
    const int dc = static_cast<int>(static_cast<uint64_t>(in[0]) << 2);
#pragma unroll
    for (int r = 0; r < 8; ++r) ws[r * 8 + col] = dc;
    return;
  }
  int64_t z2 = in[2], z3 = in[6];
  int64_t z1 = (z2 + z3) * F0541;
  int64_t tmp2 = z1 + z3 * -F1847, tmp3 = z1 + z2 * F0765;
  z2 = in[0];
  z3 = in[4];
  int64_t tmp0 = static_cast<int64_t>(static_cast<uint64_t>(z2 + z3) << 13);
  int64_t tmp1 = static_cast<int64_t>(static_cast<uint64_t>(z2 - z3) << 13);
  const int64_t tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  tmp0 = in[7];
  tmp1 = in[5];
  tmp2 = in[3];
  tmp3 = in[1];
  z1 = tmp0 + tmp3;
  z2 = tmp1 + tmp2;
  z3 = tmp0 + tmp2;
  int64_t z4 = tmp1 + tmp3;
  const int64_t z5 = (z3 + z4) * F1175;
  tmp0 *= F0298;
  tmp1 *= F2053;
  tmp2 *= F3072;
  tmp3 *= F1501;
  z1 *= -F0899;
  z2 *= -F2562;
  z3 *= -F1961;
  z4 *= -F0390;
  z3 += z5;
  z4 += z5;
  tmp0 += z1 + z3;
  tmp1 += z2 + z4;
  tmp2 += z2 + z3;
  tmp3 += z1 + z4;
  constexpr int S = 13 - 2;
  constexpr int64_t R = int64_t(1) << (S - 1);
  ws[0 * 8 + col] = static_cast<int>((tmp10 + tmp3 + R) >> S);
  ws[7 * 8 + col] = static_cast<int>((tmp10 - tmp3 + R) >> S);
  ws[1 * 8 + col] = static_cast<int>((tmp11 + tmp2 + R) >> S);
  ws[6 * 8 + col] = static_cast<int>((tmp11 - tmp2 + R) >> S);
  ws[2 * 8 + col] = static_cast<int>((tmp12 + tmp1 + R) >> S);
  ws[5 * 8 + col] = static_cast<int>((tmp12 - tmp1 + R) >> S);
  ws[3 * 8 + col] = static_cast<int>((tmp13 + tmp0 + R) >> S);
  ws[4 * 8 + col] = static_cast<int>((tmp13 - tmp0 + R) >> S);
}

Y3J_HD void idct_row(const int* ws, int row, uint8_t* out) {
  const int* w = ws + row * 8;
  constexpr int S = 13 + 2 + 3;
  constexpr int64_t R = int64_t(1) << (S - 1);
  if (w[1] == 0 && w[2] == 0 && w[3] == 0 && w[4] == 0 && w[5] == 0 && w[6] == 0 && w[7] == 0) {
    const uint8_t dc = static_cast<uint8_t>(range_limit((static_cast<int64_t>(w[0]) + 16) >> 5));
#pragma unroll
    for (int k = 0; k < 8; ++k) out[k] = dc;
    return;
  }
  int64_t z2 = w[2], z3 = w[6];
  int64_t z1 = (z2 + z3) * F0541;
  int64_t tmp2 = z1 + z3 * -F1847, tmp3 = z1 + z2 * F0765;
  int64_t tmp0 = static_cast<int64_t>(static_cast<uint64_t>(static_cast<int64_t>(w[0]) + w[4]) << 13);
  int64_t tmp1 = static_cast<int64_t>(static_cast<uint64_t>(static_cast<int64_t>(w[0]) - w[4]) << 13);
  const int64_t tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  tmp0 = w[7];
  tmp1 = w[5];
  tmp2 = w[3];
  tmp3 = w[1];
  z1 = tmp0 + tmp3;
  z2 = tmp1 + tmp2;
  z3 = tmp0 + tmp2;
  int64_t z4 = tmp1 + tmp3;
  const int64_t z5 = (z3 + z4) * F1175;
  tmp0 *= F0298;
  tmp1 *= F2053;
  tmp2 *= F3072;
  tmp3 *= F1501;
  z1 *= -F0899;
  z2 *= -F2562;
  z3 *= -F1961;
  z4 *= -F0390;
  z3 += z5;
  z4 += z5;
  tmp0 += z1 + z3;
  tmp1 += z2 + z4;
  tmp2 += z2 + z3;
  tmp3 += z1 + z4;
  out[0] = static_cast<uint8_t>(range_limit((tmp10 + tmp3 + R) >> S));
  out[7] = static_cast<uint8_t>(range_limit((tmp10 - tmp3 + R) >> S));
  out[1] = static_cast<uint8_t>(range_limit((tmp11 + tmp2 + R) >> S));
  out[6] = static_cast<uint8_t>(range_limit((tmp11 - tmp2 + R) >> S));
  out[2] = static_cast<uint8_t>(range_limit((tmp12 + tmp1 + R) >> S));
  out[5] = static_cast<uint8_t>(range_limit((tmp12 - tmp1 + R) >> S));
  out[3] = static_cast<uint8_t>(range_limit((tmp13 + tmp0 + R) >> S));
  out[4] = static_cast<uint8_t>(range_limit((tmp13 - tmp0 + R) >> S));
}

// where DCT block `blk` (MCU order) lands: component and its top-left sample in that component's plane
Y3J_HD void block_place(const y3_jpeg_geom& g, int blk, int& c, int& bx, int& by) {
  const int mcu = blk / g.blocks_per_mcu, b = blk - mcu * g.blocks_per_mcu;
  const int mx = mcu % g.mcus_x, my = mcu / g.mcus_x;
  c = mcu_comp(g, b);
  const int hc = c == 0 ? g.hmax : 1, vc = c == 0 ? g.vmax : 1;
  const int k = c == 0 ? b : 0;
  bx = (mx * hc + k % hc) * 8;
  by = (my * vc + k / hc) * 8;
}

// ------------------------------------------------------------------------------- upsample, colour, orientation, store
Y3J_HD int clamp255(int v) { return v < 0 ? 0 : (v > 255 ? 255 : v); }

// chroma sample of plane P (real size cw x ch, row pitch pitch) at full-resolution pixel (x, y)
Y3J_HD int chroma_at(const y3_jpeg_geom& g, const uint8_t* P, int pitch, int cw, int ch, int x, int y) {
  if (g.hmax == 1 && g.vmax == 1) return P[static_cast<int64_t>(y) * pitch + x];
  if (g.hmax == 4) return P[static_cast<int64_t>(y) * pitch + (x >> 2)];
  if (g.hmax == 2 && cw <= 2) return P[static_cast<int64_t>(y / g.vmax) * pitch + (x >> 1)];
  if (g.vmax == 1) {  // h2v1
    const uint8_t* row = P + static_cast<int64_t>(y) * pitch;
    const int i = x >> 1;
    return (x & 1) ? (3 * row[i] + row[i + 1 < cw ? i + 1 : i] + 2) >> 2 : (3 * row[i] + row[i > 0 ? i - 1 : 0] + 1) >> 2;
  }
  const int j = y >> 1;
  const int jn = (y & 1) ? (j + 1 < ch ? j + 1 : j) : (j > 0 ? j - 1 : 0);
  const uint8_t* r0 = P + static_cast<int64_t>(j) * pitch;
  const uint8_t* r1 = P + static_cast<int64_t>(jn) * pitch;
  if (g.hmax == 1)  // h1v2
    return (3 * r0[x] + r1[x] + ((y & 1) ? 2 : 1)) >> 2;
  const int i = x >> 1;  // h2v2
  const int cs = 3 * r0[i] + r1[i];
  if (x & 1) {
    const int n = i + 1 < cw ? i + 1 : i;
    return (3 * cs + 3 * r0[n] + r1[n] + 7) >> 4;
  }
  const int pv = i > 0 ? i - 1 : 0;
  return (3 * cs + 3 * r0[pv] + r1[pv] + 8) >> 4;
}

// output pixel (ox, oy) of the oriented image -> BGR
Y3J_HD void pixel_bgr(const y3_jpeg_geom& g, const uint8_t* const* planes, const int32_t* pitch, int ox, int oy,
                      uint8_t* bgr) {
  const int H = g.src_h, W = g.src_w;
  int x = ox, y = oy;
  switch (g.orientation) {
    case 2: x = W - 1 - ox; break;
    case 3: x = W - 1 - ox; y = H - 1 - oy; break;
    case 4: y = H - 1 - oy; break;
    case 5: x = oy; y = ox; break;
    case 6: x = oy; y = H - 1 - ox; break;
    case 7: x = W - 1 - oy; y = H - 1 - ox; break;
    case 8: x = W - 1 - oy; y = ox; break;
    default: break;
  }
  const int Y = planes[0][static_cast<int64_t>(y) * pitch[0] + x];
  if (g.ncomp == 1) {
    bgr[0] = bgr[1] = bgr[2] = static_cast<uint8_t>(Y);
    return;
  }
  const int cw = (W + g.hmax - 1) / g.hmax, ch = (H + g.vmax - 1) / g.vmax;
  const int cb = chroma_at(g, planes[1], pitch[1], cw, ch, x, y) - 128;
  const int cr = chroma_at(g, planes[2], pitch[2], cw, ch, x, y) - 128;
  const int r = Y + ((91881 * cr + 32768) >> 16);
  const int gg = Y + ((-46802 * cr - 22554 * cb + 32768) >> 16);
  const int b = Y + ((116130 * cb + 32768) >> 16);
  bgr[0] = static_cast<uint8_t>(clamp255(b));
  bgr[1] = static_cast<uint8_t>(clamp255(gg));
  bgr[2] = static_cast<uint8_t>(clamp255(r));
}

// ---------------------------------------------------------------------------------------------------- host parse
struct Reader {
  const uint8_t* d;
  int64_t n, i;
  int u16(int64_t at) const { return d[at] << 8 | d[at + 1]; }
};

inline bool build_huff(const uint8_t* bits, const uint8_t* vals, int nvals, bool dc, Huff& h) {
  memset(&h, 0, sizeof(h));
  int size[257], code[256];
  int p = 0;
  for (int l = 1; l <= 16; ++l)
    for (int i = 0; i < bits[l - 1]; ++i) size[p++] = l;
  size[p] = 0;
  if (p != nvals) return false;
  int c = 0, si = size[0];
  p = 0;
  while (size[p]) {
    while (size[p] == si) code[p++] = c++;
    if (c >= (1 << si)) return false;
    c <<= 1;
    ++si;
  }
  p = 0;
  for (int l = 1; l <= 16; ++l) {
    if (bits[l - 1]) {
      h.valoff[l] = p - code[p];
      p += bits[l - 1];
      h.maxcode[l] = code[p - 1];
    } else {
      h.maxcode[l] = -1;
    }
  }
  h.maxcode[17] = 0xFFFFF;
  h.maxcode[0] = -1;
  for (int i = 0; i < nvals; ++i) {
    h.vals[i] = vals[i];
    if (dc && vals[i] > 15) return false;
  }
  p = 0;
  for (int l = 1; l <= 9; ++l)
    for (int i = 0; i < bits[l - 1]; ++i, ++p) {
      const int base = code[p] << (9 - l);
      for (int k = 0; k < (1 << (9 - l)); ++k) h.lut[base + k] = static_cast<uint16_t>(l << 8 | vals[p]);
    }
  return true;
}

// EXIF orientation of an APP1 payload that starts "Exif\0\0": 1-8, 1 if absent, 0 if the block cannot be read
inline int exif_orientation(const uint8_t* e, int64_t n) {
  if (n < 14) return 0;
  const uint8_t* t = e + 6;
  const int64_t tn = n - 6;
  bool le;
  if (t[0] == 'I' && t[1] == 'I') le = true;
  else if (t[0] == 'M' && t[1] == 'M') le = false;
  else return 0;
  auto rd16 = [&](int64_t at) -> int { return le ? (t[at] | t[at + 1] << 8) : (t[at] << 8 | t[at + 1]); };
  auto rd32 = [&](int64_t at) -> int64_t {
    return le ? (int64_t(t[at]) | int64_t(t[at + 1]) << 8 | int64_t(t[at + 2]) << 16 | int64_t(t[at + 3]) << 24)
              : (int64_t(t[at]) << 24 | int64_t(t[at + 1]) << 16 | int64_t(t[at + 2]) << 8 | int64_t(t[at + 3]));
  };
  if (rd16(2) != 42) return 0;
  const int64_t ifd = rd32(4);
  if (ifd < 8 || ifd + 2 > tn) return 0;
  const int cnt = rd16(ifd);
  if (ifd + 2 + 12 * int64_t(cnt) > tn) return 0;
  for (int k = 0; k < cnt; ++k) {
    const int64_t at = ifd + 2 + 12 * int64_t(k);
    if (rd16(at) == 0x0112) {
      const int v = rd16(at + 8);
      if (rd16(at + 2) != 3 || rd32(at + 4) != 1 || v < 1 || v > 8) return 0;
      return v;
    }
  }
  return 1;
}

// see y3_jpeg_parse in include/yolov3_b200.h
inline void parse(const uint8_t* d, int64_t n, y3_jpeg_info* info, int32_t* segs, int32_t seg_cap) {
  memset(info, 0, sizeof(*info));
  y3_jpeg_geom& g = info->geom;
  Tables& T = *reinterpret_cast<Tables*>(info->tables);
  uint8_t hbits[8][16], hvals[8][256];
  int hn[8] = {0};
  bool hdef[8] = {false};
  uint16_t qt[4][64];
  bool qdef[4] = {false};
  int comp_id[3] = {0}, comp_hv[3] = {0}, comp_tq[3] = {0};
  int ri = 0, orientation = 1, adobe = -1, n_app1 = 0;
  bool sof = false;
  uint8_t nat[64];
  zigzag_table(nat);
  if (n < 4 || d[0] != 0xFF || d[1] != 0xD8) return;
  int64_t i = 2;
  for (;;) {
    if (i + 1 >= n || d[i] != 0xFF) return;
    while (i < n && d[i] == 0xFF) ++i;
    if (i >= n) return;
    const int m = d[i++];
    if (m == 0xD9 || m == 0x01 || (m >= 0xD0 && m <= 0xD7)) return;  // EOI before the scan, TEM, stray RST
    if (i + 2 > n) return;
    const int len = d[i] << 8 | d[i + 1];
    if (len < 2 || i + len > n) return;
    const uint8_t* s = d + i + 2;
    const int sl = len - 2;
    if (m == 0xC0 || m == 0xC1) {
      if (sof || sl < 6 || s[0] != 8) return;
      sof = true;
      g.src_h = s[1] << 8 | s[2];
      g.src_w = s[3] << 8 | s[4];
      g.ncomp = s[5];
      if (g.src_h < 1 || g.src_w < 1 || (g.ncomp != 1 && g.ncomp != 3) || sl != 6 + 3 * g.ncomp) return;
      for (int c = 0; c < g.ncomp; ++c) {
        comp_id[c] = s[6 + 3 * c];
        comp_hv[c] = s[7 + 3 * c];
        comp_tq[c] = s[8 + 3 * c];
        if (comp_tq[c] > 3) return;
      }
    } else if ((m >= 0xC2 && m <= 0xCF && m != 0xC4) || m == 0xDC || m == 0xDE || m == 0xDF) {
      return;  // progressive, lossless, arithmetic, hierarchical, DNL
    } else if (m == 0xC4) {
      int o = 0;
      while (o < sl) {
        if (o + 17 > sl) return;
        const int tc = s[o] >> 4, th = s[o] & 15;
        if (tc > 1 || th > 3) return;
        int cnt = 0;
        for (int l = 0; l < 16; ++l) cnt += s[o + 1 + l];
        if (cnt > 256 || o + 17 + cnt > sl) return;
        const int k = tc * 4 + th;
        memcpy(hbits[k], s + o + 1, 16);
        memcpy(hvals[k], s + o + 17, cnt);
        hn[k] = cnt;
        hdef[k] = true;
        o += 17 + cnt;
      }
    } else if (m == 0xDB) {
      int o = 0;
      while (o < sl) {
        const int pq = s[o] >> 4, tq = s[o] & 15;
        if (pq > 1 || tq > 3 || o + 1 + 64 * (pq + 1) > sl) return;
        for (int k = 0; k < 64; ++k) {
          const int v = pq ? (s[o + 1 + 2 * k] << 8 | s[o + 2 + 2 * k]) : s[o + 1 + k];
          if (v > 32767) return;
          qt[tq][nat[k]] = static_cast<uint16_t>(v);
        }
        qdef[tq] = true;
        o += 1 + 64 * (pq + 1);
      }
    } else if (m == 0xDD) {
      if (sl < 2) return;
      ri = s[0] << 8 | s[1];
    } else if (m == 0xE1) {
      ++n_app1;
      if (sl >= 6 && memcmp(s, "Exif\0\0", 6) == 0) {
        if (n_app1 != 1) return;  // an EXIF block behind another APP1: leave it to the host decoder
        orientation = exif_orientation(s, sl);
        if (orientation == 0) return;
      }
    } else if (m == 0xEE) {
      if (sl >= 12 && memcmp(s, "Adobe", 5) == 0) adobe = s[11];
    } else if (m == 0xDA) {
      if (!sof || sl < 1 || s[0] != g.ncomp || sl != 4 + 2 * g.ncomp) return;
      for (int c = 0; c < g.ncomp; ++c) {
        if (s[1 + 2 * c] != comp_id[c]) return;
        g.comp_dc[c] = s[2 + 2 * c] >> 4;
        g.comp_ac[c] = s[2 + 2 * c] & 15;
        if (g.comp_dc[c] > 1 || g.comp_ac[c] > 1) return;
        if (!hdef[g.comp_dc[c]] || !hdef[4 + g.comp_ac[c]] || !qdef[comp_tq[c]]) return;
      }
      const uint8_t* t = s + 1 + 2 * g.ncomp;
      if (t[0] != 0 || t[1] != 63 || t[2] != 0) return;
      i += len;
      break;
    }
    i += len;
  }
  // colour space and sampling
  if (g.ncomp == 3) {
    if (adobe == 0 || (comp_id[0] == 'R' && comp_id[1] == 'G' && comp_id[2] == 'B')) return;
    if (comp_hv[1] != 0x11 || comp_hv[2] != 0x11) return;
    g.hmax = comp_hv[0] >> 4;
    g.vmax = comp_hv[0] & 15;
    const int hv = g.hmax * 16 + g.vmax;
    if (hv != 0x11 && hv != 0x21 && hv != 0x22 && hv != 0x12 && hv != 0x41) return;
    g.mcus_x = (g.src_w + 8 * g.hmax - 1) / (8 * g.hmax);
    g.mcus_y = (g.src_h + 8 * g.vmax - 1) / (8 * g.vmax);
    g.blocks_per_mcu = g.hmax * g.vmax + 2;
  } else {  // one component: a non-interleaved scan, one block per MCU whatever its sampling factors
    g.hmax = g.vmax = 1;
    g.mcus_x = (g.src_w + 7) / 8;
    g.mcus_y = (g.src_h + 7) / 8;
    g.blocks_per_mcu = 1;
  }
  const int64_t mcus = int64_t(g.mcus_x) * g.mcus_y;
  if (mcus * g.blocks_per_mcu > (int64_t(1) << 30)) return;
  g.n_blocks = static_cast<int32_t>(mcus * g.blocks_per_mcu);
  g.restart_interval = ri;
  for (int c = 0; c < g.ncomp; ++c) memcpy(T.quant[c], qt[comp_tq[c]], sizeof(T.quant[c]));
  for (int k = 0; k < 2; ++k) {
    if (hdef[k] && !build_huff(hbits[k], hvals[k], hn[k], true, T.huff[k])) return;
    if (hdef[4 + k] && !build_huff(hbits[4 + k], hvals[4 + k], hn[4 + k], false, T.huff[2 + k])) return;
  }
  // the entropy-coded data: unstuffed length, restart segments, then EOI
  info->data_off = i;
  int64_t u = 0, seg_start = 0;
  int nseg = 0, next_rst = 0;
  auto add_seg = [&](int64_t end) {
    if (nseg < seg_cap) {
      segs[2 * nseg] = static_cast<int32_t>(seg_start);
      segs[2 * nseg + 1] = static_cast<int32_t>(end - seg_start);
    }
    ++nseg;
    seg_start = end;
  };
  for (;;) {
    if (i >= n) return;  // no EOI
    if (d[i] != 0xFF) { ++u; ++i; continue; }
    int64_t j = i + 1;
    while (j < n && d[j] == 0xFF) ++j;
    if (j >= n) return;
    if (d[j] == 0x00) { ++u; i = j + 1; continue; }
    const int m = d[j];
    if (m >= 0xD0 && m <= 0xD7) {
      if (!ri || m - 0xD0 != next_rst) return;  // wrong restart sequence
      next_rst = (next_rst + 1) & 7;
      add_seg(u);
      i = j + 1;
      continue;
    }
    if (m != 0xD9) return;  // another scan (multi-scan), DNL or anything else before EOI
    add_seg(u);
    g.data_len = static_cast<int32_t>(i - info->data_off);
    break;
  }
  if (u > (int64_t(1) << 27)) return;
  g.unstuffed_len = static_cast<int32_t>(u);
  g.n_segs = nseg;
  const int64_t want = ri ? (mcus + ri - 1) / ri : 1;
  if (nseg != want) return;
  g.orientation = orientation;
  g.height = orientation >= 5 ? g.src_w : g.src_h;
  g.width = orientation >= 5 ? g.src_h : g.src_w;
  info->eligible = 1;
}

}  // namespace jpeg
}  // namespace y3
