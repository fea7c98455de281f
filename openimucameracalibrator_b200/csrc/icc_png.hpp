// PNG decoding on the host for the drop-in extract_board_to_json: the pixels cv::imread(path, IMREAD_COLOR) returns (OpenCV 4.13 on
// libpng 1.6), header-only, on the system zlib (link with -lz).
//
// What imread's PNG path does, and so what this does:
//   colour types 0 (gray), 2 (RGB), 3 (palette), 4 (gray + alpha), 6 (RGBA); bit depths 1, 2, 4, 8, 16 where the format allows them;
//   all five row filters, Adam7 interlacing, IDAT split over any number of chunks;
//   16-bit samples keep their high byte (v >> 8: png_set_strip_16, not rounding and not v / 257);
//   gray below 8 bits is scaled to 0..255 (v * 255 / (2^d - 1)); palette indices are looked up, an index past the palette is black;
//   alpha and tRNS are dropped without compositing (png_set_strip_alpha), gray is replicated to B = G = R by imread -- here gray
//   images (types 0 and 4) come back as one channel, colour ones (2, 3, 6) as three in B, G, R order;
//   an eXIf orientation is applied by imread, so a file whose orientation is not 1 (top-left) is refused rather than read rotated.
// Malformed input is an error that names the file, never a crash: a bad signature, a CRC mismatch in any chunk, a missing or bad IHDR,
// a missing PLTE for a palette image, zero or absurd dimensions, an unknown critical chunk, truncated or excess IDAT data.
// Inflate and unfiltering are serial within one file; a caller decodes several files in parallel.
#pragma once
#include <zlib.h>

#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

namespace iccpng {

struct Image {
  int width = 0, height = 0, channels = 0;   // channels: 1 (gray) or 3 (B, G, R)
  std::vector<uint8_t> px;                   // height rows of width * channels bytes
};

constexpr uint32_t kMaxSide = 1u << 16;                 // larger sides are refused as absurd
constexpr uint64_t kMaxPixels = uint64_t(1) << 28;      // 268 M pixels

namespace detail {

inline uint32_t be32(const uint8_t* p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }

inline int paeth(int a, int b, int c) {
  const int p = a + b - c, pa = p > a ? p - a : a - p, pb = p > b ? p - b : b - p, pc = p > c ? p - c : c - p;
  return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

// in place: rows of `rowbytes` bytes, each after its filter byte; false for an unknown filter type
inline bool unfilter(uint8_t* data, size_t rows, size_t rowbytes, int bpp) {
  const uint8_t* prior = nullptr;
  for (size_t y = 0; y < rows; ++y) {
    const int type = data[0];
    uint8_t* x = data + 1;
    switch (type) {
      case 0: break;
      case 1: for (size_t i = bpp; i < rowbytes; ++i) x[i] = (uint8_t)(x[i] + x[i - bpp]); break;
      case 2: if (prior) for (size_t i = 0; i < rowbytes; ++i) x[i] = (uint8_t)(x[i] + prior[i]); break;
      case 3:
        for (size_t i = 0; i < rowbytes; ++i) {
          const int a = i >= (size_t)bpp ? x[i - bpp] : 0, b = prior ? prior[i] : 0;
          x[i] = (uint8_t)(x[i] + ((a + b) >> 1));
        }
        break;
      case 4:
        for (size_t i = 0; i < rowbytes; ++i) {
          const int a = i >= (size_t)bpp ? x[i - bpp] : 0, b = prior ? prior[i] : 0, c = (prior && i >= (size_t)bpp) ? prior[i - bpp] : 0;
          x[i] = (uint8_t)(x[i] + paeth(a, b, c));
        }
        break;
      default: return false;
    }
    prior = x;
    data += rowbytes + 1;
  }
  return true;
}

// the orientation tag (0x0112) of an eXIf chunk's TIFF structure; 1 when it has none or cannot be read
inline int exif_orientation(const uint8_t* p, size_t n) {
  if (n < 8) return 1;
  const bool le = p[0] == 'I' && p[1] == 'I';
  if (!le && !(p[0] == 'M' && p[1] == 'M')) return 1;
  auto u16 = [&](size_t o) -> uint32_t { return le ? (uint32_t)p[o] | (uint32_t)p[o + 1] << 8 : (uint32_t)p[o] << 8 | p[o + 1]; };
  auto u32 = [&](size_t o) -> uint32_t { return le ? u16(o) | u16(o + 2) << 16 : u16(o) << 16 | u16(o + 2); };
  const size_t ifd = u32(4);
  if (ifd + 2 > n) return 1;
  const uint32_t count = u16(ifd);
  for (uint32_t k = 0; k < count; ++k) {
    const size_t e = ifd + 2 + 12 * (size_t)k;
    if (e + 12 > n) return 1;
    if (u16(e) == 0x0112 && u16(e + 2) == 3) return (int)u16(e + 8);
  }
  return 1;
}

}  // namespace detail

// The decoded image of `data`, the bytes of the file `name` (used in messages only).  Throws std::runtime_error naming the file.
inline Image decode(const std::string& name, const uint8_t* data, size_t size) {
  auto fail = [&](const std::string& why) -> void { throw std::runtime_error(name + ": " + why); };
  static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n'};
  if (size < 8 || memcmp(data, sig, 8) != 0) fail("not a PNG file (bad signature)");
  size_t pos = 8;
  uint32_t W = 0, H = 0; int depth = 0, ctype = -1, interlace = 0;
  uint8_t palette[256][3] = {};
  int n_palette = 0;
  bool have_ihdr = false, have_plte = false, idat_done = false, have_iend = false, in_idat = false;
  std::vector<uint8_t> z;
  while (pos < size) {
    if (size - pos < 12) fail("truncated chunk");
    const uint32_t len = detail::be32(data + pos);
    if (len > 0x7fffffffu || size - pos - 12 < len) fail("truncated chunk");
    const uint8_t* type = data + pos + 4;
    const uint8_t* body = data + pos + 8;
    const std::string tname(reinterpret_cast<const char*>(type), 4);
    for (int k = 0; k < 4; ++k) if (!((type[k] >= 'A' && type[k] <= 'Z') || (type[k] >= 'a' && type[k] <= 'z'))) fail("bad chunk type");
    if ((uint32_t)crc32(crc32(0L, Z_NULL, 0), type, len + 4) != detail::be32(body + len)) fail("CRC mismatch in chunk " + tname);
    pos += 12 + (size_t)len;
    if (!have_ihdr && tname != "IHDR") fail("the first chunk is not IHDR");
    if (tname != "IDAT" && in_idat) { in_idat = false; idat_done = true; }
    if (tname == "IHDR") {
      if (have_ihdr || len != 13) fail("bad IHDR");
      have_ihdr = true;
      W = detail::be32(body); H = detail::be32(body + 4); depth = body[8]; ctype = body[9]; interlace = body[12];
      if (W == 0 || H == 0) fail("zero image width or height");
      if (W > kMaxSide || H > kMaxSide || (uint64_t)W * H > kMaxPixels) fail("image dimensions " + std::to_string(W) + " x " + std::to_string(H) + " are too large");
      const bool ok = (ctype == 0 && (depth == 1 || depth == 2 || depth == 4 || depth == 8 || depth == 16)) ||
                      (ctype == 3 && (depth == 1 || depth == 2 || depth == 4 || depth == 8)) ||
                      ((ctype == 2 || ctype == 4 || ctype == 6) && (depth == 8 || depth == 16));
      if (!ok) fail("invalid colour type " + std::to_string(ctype) + " with bit depth " + std::to_string(depth));
      if (body[10] != 0 || body[11] != 0 || interlace > 1) fail("unknown compression, filter or interlace method");
    } else if (tname == "PLTE") {
      if (have_plte || len % 3 || len == 0 || len > 768 || !z.empty()) fail("bad PLTE");
      have_plte = true;
      n_palette = (int)(len / 3);
      for (int k = 0; k < n_palette; ++k) for (int c = 0; c < 3; ++c) palette[k][c] = body[3 * k + c];
    } else if (tname == "IDAT") {
      if (idat_done) fail("IDAT chunks are not consecutive");
      in_idat = true;
      z.insert(z.end(), body, body + len);
    } else if (tname == "IEND") {
      have_iend = true;
      break;
    } else if (tname == "eXIf") {
      const int o = detail::exif_orientation(body, len);
      if (o != 1) fail("EXIF orientation " + std::to_string(o) + " is not supported (cv::imread would rotate the image)");
    } else if (!(type[0] & 0x20)) {
      fail("unknown critical chunk " + tname);
    }
  }
  if (!have_ihdr) fail("no IHDR");
  if (z.empty()) fail("no image data (IDAT)");
  if (!have_iend) fail("truncated file (no IEND)");
  if (ctype == 3 && !have_plte) fail("palette image without PLTE");
  const int ch = ctype == 0 || ctype == 3 ? 1 : ctype == 2 ? 3 : ctype == 4 ? 2 : 4;
  const int bits = ch * depth, bpp = bits >= 8 ? bits / 8 : 1;
  // Adam7 passes (or the whole image), their sizes and raw byte counts
  static const int A7[7][4] = {{0, 0, 8, 8}, {4, 0, 8, 8}, {0, 4, 4, 8}, {2, 0, 4, 4}, {0, 2, 2, 4}, {1, 0, 2, 2}, {0, 1, 1, 2}};
  struct Pass { int x0, y0, dx, dy; size_t w, h, rowbytes, offset; };
  std::vector<Pass> passes;
  size_t total = 0;
  for (int k = 0; k < (interlace ? 7 : 1); ++k) {
    Pass p{0, 0, 1, 1, W, H, 0, 0};
    if (interlace) {
      p.x0 = A7[k][0]; p.y0 = A7[k][1]; p.dx = A7[k][2]; p.dy = A7[k][3];
      p.w = W > (uint32_t)p.x0 ? (W - p.x0 + p.dx - 1) / p.dx : 0; p.h = H > (uint32_t)p.y0 ? (H - p.y0 + p.dy - 1) / p.dy : 0;
    }
    if (p.w == 0 || p.h == 0) continue;
    p.rowbytes = (p.w * bits + 7) / 8; p.offset = total;
    total += p.h * (p.rowbytes + 1);
    passes.push_back(p);
  }
  std::vector<uint8_t> raw(total + 1);
  z_stream s;
  memset(&s, 0, sizeof s);
  if (inflateInit(&s) != Z_OK) fail("zlib initialisation failed");
  s.next_in = z.data(); s.avail_in = (uInt)z.size();
  s.next_out = raw.data(); s.avail_out = (uInt)raw.size();
  const int zr = inflate(&s, Z_FINISH);
  const size_t produced = raw.size() - s.avail_out, left = s.avail_in;
  inflateEnd(&s);
  if (zr == Z_DATA_ERROR || zr == Z_NEED_DICT || zr == Z_MEM_ERROR) fail("corrupt image data (zlib: " + std::string(s.msg ? s.msg : "error") + ")");
  if (produced > total) fail("excess image data (more than the image needs)");
  if (zr != Z_STREAM_END || produced < total) fail("truncated image data");
  if (left != 0) fail("excess data after the end of the compressed image stream");
  Image img;
  img.width = (int)W; img.height = (int)H; img.channels = (ctype == 0 || ctype == 4) ? 1 : 3;
  img.px.assign((size_t)W * H * img.channels, 0);
  const int maxv = (1 << depth) - 1;
  for (const Pass& p : passes) {
    uint8_t* rows = raw.data() + p.offset;
    if (!detail::unfilter(rows, p.h, p.rowbytes, bpp)) fail("unknown row filter type");
    for (size_t y = 0; y < p.h; ++y) {
      const uint8_t* r = rows + y * (p.rowbytes + 1) + 1;
      auto sample = [&](size_t i) -> int {   // sample i of the row, scaled to 8 bits as imread does (palette indices stay indices)
        if (depth == 8) return r[i];
        if (depth == 16) return r[2 * i];
        const int v = (r[(i * depth) >> 3] >> (8 - depth - (int)((i * depth) & 7))) & maxv;
        return ctype == 3 ? v : v * 255 / maxv;
      };
      uint8_t* out = img.px.data() + ((size_t)(p.y0 + y * p.dy) * W) * img.channels;
      for (size_t x = 0; x < p.w; ++x) {
        uint8_t* o = out + (size_t)(p.x0 + x * p.dx) * img.channels;
        switch (ctype) {
          case 0: case 4: o[0] = (uint8_t)sample(x * ch); break;
          case 2: case 6: o[0] = (uint8_t)sample(x * ch + 2); o[1] = (uint8_t)sample(x * ch + 1); o[2] = (uint8_t)sample(x * ch); break;
          case 3: {
            const int k = sample(x);
            if (k < n_palette) { o[0] = palette[k][2]; o[1] = palette[k][1]; o[2] = palette[k][0]; }
            break;
          }
        }
      }
    }
  }
  return img;
}

inline Image decode_file(const std::string& path) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) throw std::runtime_error(path + ": cannot open");
  std::vector<uint8_t> buf;
  uint8_t tmp[1 << 16];
  size_t n;
  while ((n = fread(tmp, 1, sizeof tmp, f)) > 0) buf.insert(buf.end(), tmp, tmp + n);
  const bool err = ferror(f) != 0;
  fclose(f);
  if (err) throw std::runtime_error(path + ": read error");
  return decode(path, buf.data(), buf.size());
}

}  // namespace iccpng
