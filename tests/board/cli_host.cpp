// Host-side test shim for the host code of the drop-in extract_board_to_json: the PNG decoder (csrc/icc_png.hpp), the UBJSON writer
// (csrc/icc_json.hpp) and the corner-file board reader (csrc/icc_cli_common.hpp), compiled with g++ -lz for the `-m "not gpu"` suite.
#include "../../openimucameracalibrator_b200/csrc/icc_cli_common.hpp"
#include "../../openimucameracalibrator_b200/csrc/icc_png.hpp"

#include <cstring>
#include <string>

namespace {
std::string g_error;
iccpng::Image g_image;
std::string g_bytes;
std::vector<double> g_board;
}

extern "C" {
// decodes `size` bytes; 1 on success (read the result with png_result), 0 with the message in last_error
int png_decode(const uint8_t* data, size_t size, int* width, int* height, int* channels) {
  try {
    g_image = iccpng::decode("test.png", data, size);
    *width = g_image.width; *height = g_image.height; *channels = g_image.channels;
    return 1;
  } catch (const std::exception& e) { g_error = e.what(); return 0; }
}
void png_result(uint8_t* out) { memcpy(out, g_image.px.data(), g_image.px.size()); }
const char* last_error() { return g_error.c_str(); }
// text JSON -> UBJSON bytes as the CLI writes them; returns the byte count (-1 on a parse error), copy them with bytes_result
long long ubjson_from_text(const char* text) {
  try { g_bytes = iccjson::dump_ubjson(iccjson::parse_text(text)); return (long long)g_bytes.size(); }
  catch (const std::exception& e) { g_error = e.what(); return -1; }
}
void bytes_result(uint8_t* out) { memcpy(out, g_bytes.data(), g_bytes.size()); }
// UBJSON corner file -> icccli::read_scene_points; returns the point count (-1 on an error), copy 4 doubles per point with board_result
int scene_points(const uint8_t* data, size_t size) {
  try {
    const std::string d(reinterpret_cast<const char*>(data), size);
    int n = 0;
    g_board = icccli::read_scene_points(iccjson::UbjsonParser(d).parse(), n);
    return n;
  } catch (const std::exception& e) { g_error = e.what(); return -1; }
}
void board_result(double* out) { memcpy(out, g_board.data(), g_board.size() * sizeof(double)); }
}
