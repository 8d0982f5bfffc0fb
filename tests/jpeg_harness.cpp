// Host emulation of the device JPEG decode (csrc/y3_jpeg.cu): the same per-thread steps from csrc/y3_jpeg.cuh, run in the
// kernels' phase order.  Built with g++ by tests/test_jpeg_cpu.py.  Usage: jpeg_harness in.jpg out.bin
// out.bin: int32 eligible, err, height, width, then height * width * 3 BGR bytes (when eligible).
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../yolov3_b200/csrc/y3_jpeg.cuh"

using namespace y3::jpeg;

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 2;
  std::vector<uint8_t> buf;
  uint8_t tmp[65536];
  size_t k;
  while ((k = fread(tmp, 1, sizeof(tmp), f)) > 0) buf.insert(buf.end(), tmp, tmp + k);
  fclose(f);
  static y3_jpeg_info info;
  std::vector<int32_t> segs(2 * 16);
  parse(buf.data(), static_cast<int64_t>(buf.size()), &info, segs.data(), 16);
  if (info.eligible && info.geom.n_segs > 16) {
    segs.resize(2 * info.geom.n_segs);
    parse(buf.data(), static_cast<int64_t>(buf.size()), &info, segs.data(), info.geom.n_segs);
  }
  FILE* o = fopen(argv[2], "wb");
  const y3_jpeg_geom& g = info.geom;
  int32_t hdr[4] = {info.eligible, 0, g.height, g.width};
  if (!info.eligible) {
    fwrite(hdr, 4, 4, o);
    fclose(o);
    return 0;
  }
  const Tables& T = *reinterpret_cast<const Tables*>(info.tables);
  uint8_t nat[64];
  zigzag_table(nat);
  uint8_t canon[8];
  for (int b = 0; b < g.blocks_per_mcu; ++b) canon[b] = static_cast<uint8_t>(canonical_block(g, b));
  // 1. unstuff
  const uint8_t* data = buf.data() + info.data_off;
  std::vector<uint8_t> un(g.unstuffed_len + 8, 0);
  int u = 0;
  for (int i = 0; i < g.data_len; ++i)
    if (keep_byte(data, i, g.data_len)) un[u++] = data[i];
  int err = u != g.unstuffed_len;
  // 2. subsequences of every segment, synchronised by rounds
  std::vector<int> sub_seg, sub_idx, first;
  for (int s = 0; s < g.n_segs; ++s) {
    const int nsub = std::max(1, segs[2 * s + 1] * 8 / kSubBits);
    for (int i = 0; i < nsub; ++i) {
      sub_seg.push_back(s);
      sub_idx.push_back(i);
    }
  }
  const int n_sub = static_cast<int>(sub_seg.size());
  auto sub_args = [&](int q, int& end, bool& last) {
    const int s = sub_seg[q], nb = segs[2 * s + 1];
    const int nsub = std::max(1, nb * 8 / kSubBits);
    last = sub_idx[q] == nsub - 1;
    end = last ? nb * 8 : (sub_idx[q] + 1) * kSubBits;
  };
  std::vector<uint64_t> entry(n_sub), exitv(n_sub);
  std::vector<int> cnt(n_sub), ferr(n_sub), dirty(n_sub, 1);
  for (int q = 0; q < n_sub; ++q) entry[q] = pack_state(sub_idx[q] * kSubBits, 0, 0);
  for (int round = 0;; ++round) {
    for (int q = 0; q < n_sub; ++q) {
      if (!dirty[q]) continue;
      int end;
      bool last;
      sub_args(q, end, last);
      const int s = sub_seg[q];
      SubResult r = decode_sub<false>(g, T, nat, canon, un.data() + segs[2 * s], segs[2 * s + 1], end, last, entry[q], nullptr, 0);
      exitv[q] = r.exit;
      cnt[q] = r.blocks;
      ferr[q] = r.err;
      dirty[q] = 0;
    }
    bool changed = false;
    for (int q = 1; q < n_sub; ++q)
      if (sub_idx[q] && entry[q] != exitv[q - 1]) {
        entry[q] = exitv[q - 1];
        dirty[q] = 1;
        changed = true;
      }
    if (!changed) break;
  }
  // 3. block index of each subsequence, counts checked per segment
  std::vector<int> blk0(n_sub);
  int acc = 0;
  for (int q = 0; q < n_sub; ++q) {
    blk0[q] = acc;
    acc += cnt[q];
    err |= ferr[q];
    if (sub_idx[q] == 0 && g.restart_interval &&
        static_cast<int64_t>(blk0[q]) != static_cast<int64_t>(sub_seg[q]) * g.restart_interval * g.blocks_per_mcu)
      err = 1;
  }
  if (acc != g.n_blocks) err = 1;
  std::vector<int16_t> coef(static_cast<size_t>(g.n_blocks) * 64, 0x5a5a);
  if (!err)
    for (int q = 0; q < n_sub; ++q) {
      int end;
      bool last;
      sub_args(q, end, last);
      const int s = sub_seg[q];
      decode_sub<true>(g, T, nat, canon, un.data() + segs[2 * s], segs[2 * s + 1], end, last, entry[q], coef.data(), blk0[q]);
    }
  hdr[1] = err;
  fwrite(hdr, 4, 4, o);
  if (err) {
    fclose(o);
    return 0;
  }
  // 4. DC prediction per component, reset at each restart (wrapping, stored as 16 bits)
  const int mcus = g.mcus_x * g.mcus_y;
  for (int c = 0; c < g.ncomp; ++c) {
    const int per = c == 0 ? g.hmax * g.vmax : 1, off = c == 0 ? 0 : g.hmax * g.vmax + c - 1;
    unsigned run = 0;
    for (int i = 0; i < mcus * per; ++i) {
      const int mcu = i / per, kk = i % per;
      if (kk == 0 && (g.restart_interval ? mcu % g.restart_interval == 0 : mcu == 0)) run = 0;
      int16_t* dc = &coef[(static_cast<size_t>(mcu) * g.blocks_per_mcu + off + kk) * 64];
      run += static_cast<unsigned>(static_cast<int>(*dc));
      *dc = static_cast<int16_t>(run);
    }
  }
  // 5. IDCT into the component planes
  Layout L = layout(g);
  std::vector<std::vector<uint8_t>> planes(3);
  for (int c = 0; c < g.ncomp; ++c) planes[c].assign(static_cast<size_t>(L.pitch[c]) * L.rows[c], 0);
  for (int b = 0; b < g.n_blocks; ++b) {
    int c, bx, by;
    block_place(g, b, c, bx, by);
    int ws[64];
    for (int col = 0; col < 8; ++col) idct_col(&coef[static_cast<size_t>(b) * 64], T.quant[c], col, ws);
    for (int row = 0; row < 8; ++row) idct_row(ws, row, &planes[c][static_cast<size_t>(by + row) * L.pitch[c] + bx]);
  }
  // 6. upsample, colour, orientation
  const uint8_t* pp[3] = {planes[0].data(), g.ncomp == 3 ? planes[1].data() : nullptr,
                          g.ncomp == 3 ? planes[2].data() : nullptr};
  std::vector<uint8_t> out(static_cast<size_t>(g.height) * g.width * 3);
  for (int y = 0; y < g.height; ++y)
    for (int x = 0; x < g.width; ++x) pixel_bgr(g, pp, L.pitch, x, y, &out[(static_cast<size_t>(y) * g.width + x) * 3]);
  fwrite(out.data(), 1, out.size(), o);
  fclose(o);
  return 0;
}
