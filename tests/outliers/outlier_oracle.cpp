// Oracle of the outlier-corner rejection between spline solves (icc_get_corner_errors, icc_reject_outlier_corners, icc_get_corner_status),
// for tests/test_outlier_corners.py.
//
// oracle/icc_oracle.cpp stays as it is.  This file compiles it once more through tests/omni_radtan/omni_oracle.cpp with -DOMNI_TANGENT, so that
// the library has every camera model (omni-radtan included) and the tangent reprojection error (icco_set_tangent_bearings), and adds the
// three entry points with the product's shapes.  They state the rule over the oracle's own vision blocks:
//   * a corner's error is |(rx, ry)| of its pair from eval_block (the functor the oracle evaluates, pixel or tangent);
//   * rx == 0 || ry == 0: neither counted nor rejected; the 1e10 pair of a failed projection: not counted, always rejected;
//   * threshold = max(min_px, k_sigma sqrt(sum e^2 / count)); a corner with e > threshold leaves its block.
// Rejection rewrites the oracle's corner arrays (and bearings) with the kept corners of every frame packed in frame order, rebuilds the
// vision blocks from them and shifts the IMU blocks' residual offsets.  The arrays as icco_set_frames gave them are kept aside and put back
// by the next icco_batch_init_spline, which so reassembles from the inputs, as the product does.
#include <cmath>
#include <map>
#include <utility>
#include <vector>

#define icco_batch_init_spline(...) icco_batch_init_spline_base(__VA_ARGS__)
#define icco_set_frames(...) icco_set_frames_base(__VA_ARGS__)
#define OMNI_TANGENT
#include "../omni_radtan/omni_oracle.cpp"
#undef icco_batch_init_spline
#undef icco_set_frames

namespace {

struct Rejection {
  std::vector<double> uv, b; std::vector<int> pid, ok;   // the corner arrays of icco_set_frames (and their bearings)
  bool had_bearings = false;
  std::vector<std::pair<int, int>> ranges;               // input corner range of every frame in the problem
  std::vector<int> src;                                  // input index of every corner now in the problem, in order
};
std::map<const Oracle*, Rejection> g_rejection;

void restore_inputs(Oracle& o) {
  const auto it = g_rejection.find(&o);
  if (it == g_rejection.end()) return;
  Rejection& R = it->second;
  o.uv = R.uv; o.point_ids = R.pid;
  if (R.had_bearings) { const auto t = g_tangent.find(&o); if (t != g_tangent.end()) { t->second.b = R.b; t->second.ok = R.ok; } }
  g_rejection.erase(it);
}

bool pair_is_zero(double rx, double ry) { return rx == 0.0 || ry == 0.0; }
bool pair_failed(double rx, double ry) { return rx == 1e10 && ry == 1e10; }

// e and the pair of every corner of the problem, in frame order
void corner_pairs(Oracle& o, std::vector<double>& res) {
  res.clear();
  Scratch s;
  for (const auto& b : o.vis_blocks) { int nc; eval_block(o, b, s, false, nc); res.insert(res.end(), s.res.begin(), s.res.end()); }
}

icc_status reject(Oracle& o, double thr, double rms, double n_failed, icc_outlier_summary* out) {
  std::vector<double> res; corner_pairs(o, res);
  const int nf = int(o.frames.size());
  if (g_rejection.find(&o) == g_rejection.end()) {   // first rejection since batch_init: keep the inputs, and where each corner came from
    Rejection& R = g_rejection[&o];
    R.uv = o.uv; R.pid = o.point_ids;
    const auto t = g_tangent.find(&o);
    R.had_bearings = t != g_tangent.end();
    if (R.had_bearings) { R.b = t->second.b; R.ok = t->second.ok; }
    for (const auto& f : o.frames) { R.ranges.push_back({f.c0, f.c1}); for (int c = f.c0; c < f.c1; ++c) R.src.push_back(c); }
  }
  Rejection& R = g_rejection[&o];
  const auto t = g_tangent.find(&o);
  std::vector<double> uv(o.uv), b; std::vector<int> pid(o.point_ids), ok, src;
  if (t != g_tangent.end()) { b = t->second.b; ok = t->second.ok; }
  int pos = 0, k = 0, emptied = 0;
  const int n_before = int(res.size() / 2);
  for (int fi = 0; fi < nf; ++fi) {
    Frame& f = o.frames[fi];
    const int c0 = pos;
    for (int c = f.c0; c < f.c1; ++c, ++k) {
      const double rx = res[2 * size_t(k)], ry = res[2 * size_t(k) + 1];
      const bool keep = pair_is_zero(rx, ry) || (!pair_failed(rx, ry) && !(std::sqrt(rx * rx + ry * ry) > thr));
      if (!keep) continue;
      uv[2 * size_t(pos)] = o.uv[2 * size_t(c)]; uv[2 * size_t(pos) + 1] = o.uv[2 * size_t(c) + 1]; pid[pos] = o.point_ids[c];
      if (t != g_tangent.end()) { for (int d = 0; d < 3; ++d) b[3 * size_t(pos) + d] = t->second.b[3 * size_t(c) + d]; ok[pos] = t->second.ok[c]; }
      src.push_back(R.src[k]);
      ++pos;
    }
    if (f.c1 > f.c0 && pos == c0) ++emptied;
    f.c0 = c0; f.c1 = pos;
  }
  o.uv.swap(uv); o.point_ids.swap(pid); R.src.swap(src);
  if (t != g_tangent.end()) { t->second.b.swap(b); t->second.ok.swap(ok); }
  // vision blocks from the kept corners; the IMU blocks follow the vision residuals
  const bool rolling = o.ip.init_line_delay_s != 0.0;
  int res_vis = 0;
  for (int fi = 0; fi < nf; ++fi) {
    Block& blk = o.vis_blocks[fi];
    const Frame& f = o.frames[fi];
    blk.params.resize(2 * SPLINE_N + 3);
    for (int c = f.c0; c < f.c1; ++c) blk.params.push_back({&o.points[4 * size_t(o.point_ids[c])], 4, LP_NONE, -1});
    blk.n_res = 2 * (f.c1 - f.c0); blk.res_off = res_vis; res_vis += blk.n_res;
  }
  if (rolling) {
    for (int fi = 0; fi < nf; ++fi) o.blocks[fi] = o.vis_blocks[fi];
    int off = res_vis;
    for (size_t i = nf; i < o.blocks.size(); ++i) { o.blocks[i].res_off = off; off += o.blocks[i].n_res; }
    o.n_res_vis = res_vis;
  }
  o.cur_flags = -1;
  if (out) {
    out->n_corners = n_before; out->n_rejected = n_before - pos; out->n_failed = int64_t(n_failed); out->n_frames_emptied = emptied;
    out->rms_px = rms; out->threshold_px = thr;
  }
  return ICC_OK;
}

}  // namespace

extern "C" {

icc_status icco_set_frames(void* h, int nf, const double* t, const int32_t* off, const int32_t* ids, const double* uv, const double* q, const double* p) {
  g_rejection.erase(O(h));
  return icco_set_frames_base(h, nf, t, off, ids, uv, q, p);
}
icc_status icco_batch_init_spline(void* h, const icc_init_params* ipp) {
  restore_inputs(*O(h));
  return icco_batch_init_spline_base(h, ipp);
}

icc_status icco_get_corner_errors(void* h, int n, double* err) {
  Oracle& o = *O(h);
  if (!o.initialised) { o.err = "batch_init_spline first"; return ICC_ERR_STATE; }
  std::vector<double> res; corner_pairs(o, res);
  if (!err || size_t(n) * 2 != res.size()) { o.err = "n must be the number of corners in the solve"; return ICC_ERR_INVALID_ARGUMENT; }
  for (int c = 0; c < n; ++c) err[c] = std::sqrt(res[2 * size_t(c)] * res[2 * size_t(c)] + res[2 * size_t(c) + 1] * res[2 * size_t(c) + 1]);
  return ICC_OK;
}

icc_status icco_reject_outlier_corners(void* h, double k_sigma, double min_px, icc_outlier_summary* out) {
  Oracle& o = *O(h);
  if (!(k_sigma > 0.0) || !std::isfinite(k_sigma) || !(min_px >= 0.0) || !std::isfinite(min_px)) { o.err = "bad k_sigma / min_px"; return ICC_ERR_INVALID_ARGUMENT; }
  if (!o.initialised) { o.err = "batch_init_spline first"; return ICC_ERR_STATE; }
  std::vector<double> res; corner_pairs(o, res);
  double s2 = 0.0, cnt = 0.0, failed = 0.0;
  for (size_t c = 0; c < res.size() / 2; ++c) {
    const double rx = res[2 * c], ry = res[2 * c + 1];
    if (pair_is_zero(rx, ry)) continue;
    if (pair_failed(rx, ry)) { failed += 1.0; continue; }
    s2 += rx * rx + ry * ry; cnt += 1.0;
  }
  const double rms = cnt > 0.0 ? std::sqrt(s2 / cnt) : 0.0;
  return reject(o, std::max(min_px, k_sigma * rms), rms, failed, out);
}

// test hook: the rejection with a given threshold (shards whose sums were added up by the caller)
icc_status icco_reject_outlier_corners_at(void* h, double threshold_px, icc_outlier_summary* out) {
  Oracle& o = *O(h);
  if (!o.initialised) { o.err = "batch_init_spline first"; return ICC_ERR_STATE; }
  return reject(o, threshold_px, 0.0, 0.0, out);
}

icc_status icco_get_corner_status(const void* h, int n_input, int32_t* status) {
  const Oracle& o = *O(h);
  if (!o.initialised) return ICC_ERR_STATE;
  const auto it = g_rejection.find(&o);
  const int n_in = it != g_rejection.end() ? int(it->second.pid.size()) : int(o.point_ids.size());
  if (!status || n_input != n_in) return ICC_ERR_INVALID_ARGUMENT;
  for (int c = 0; c < n_input; ++c) status[c] = -1;
  if (it == g_rejection.end()) { for (const auto& f : o.frames) for (int c = f.c0; c < f.c1; ++c) status[c] = 1; return ICC_OK; }
  for (const auto& r : it->second.ranges) for (int c = r.first; c < r.second; ++c) status[c] = 0;
  for (const int c : it->second.src) status[c] = 1;
  return ICC_OK;
}

}  // extern "C"
