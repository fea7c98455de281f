// Drop-in host program for applications/fit_allan_variance.cc of urbste/OpenImuCameraCalibrator: the same gflags names
// (--telemetry_json, --verbose), the telemetry JSON input (timestamps ns * 1e-9 as ReadTelemetryJSON), and on stdout the lines
// AllanVarianceFitter(telemetry, 10000).RunFit() prints, in its order, with its labels and units (src/core/allan_variance_fitter.cc,
// src/allanvariance/*.cc), including its "Too few number" (fewer than 10000 samples) and "Too short time!!!!" (under 10 minutes)
// warnings.  Ceres' per-iteration progress table is not reproduced.  The computation runs on the GPU through icc_allan_variance.
// Extra flags: --device, and --output_json, which writes the curves and fits of the six channels (the reference writes no file).
#include "../../include/icc_b200.h"
#include "icc_cli_common.hpp"

#include <algorithm>
#include <fstream>
#include <iomanip>
#include <iostream>
#include <sstream>

using iccjson::Value;

namespace {
const char* kNames[6] = {"acc_x", "acc_y", "acc_z", "gyr_x", "gyr_y", "gyr_z"};
const char* kParams[5] = {"Q", "N", "B", "K", "R"};

Value array(const double* v, int n) { Value a = Value::array(); for (int i = 0; i < n; ++i) a.push_back(Value(v[i])); return a; }

// AllanGyr / AllanAcc::calc (allan_gyr.cc:35-71)
void print_calc(const std::string& name, int n, double t0, double t1, const icc_allan_summary& S) {
  std::cout << name << "  numData " << n << std::endl;
  if (n < 10000) std::cout << name << "  Too few number" << std::endl;
  std::cout << name << "  start_t " << t0 << std::endl << name << "  end_t " << t1 << std::endl;
  std::cout << name << " dt " << std::endl << "-------------" << (t1 - t0) << " s" << std::endl << "-------------" << (t1 - t0) / 60 << " min" << std::endl
            << "-------------" << (t1 - t0) / 3600 << " h" << std::endl;
  if ((t1 - t0) / 60 < 10) std::cout << name << "  Too short time!!!!" << std::endl;
  std::cout << name << "  freq " << S.freq << std::endl << name << "  period " << S.period << std::endl;
}

void print_init(const icc_allan_summary& S) {   // initValue's "C " << C.transpose(): Eigen pads every coefficient to the widest one
  size_t w = 0;
  for (int k = 0; k < 5; ++k) { std::ostringstream o; o.copyfmt(std::cout); o << S.init_coeffs[k]; w = std::max(w, o.str().size()); }
  std::cout << "C ";
  for (int k = 0; k < 5; ++k) { if (k) std::cout << " "; std::cout << std::setw((int)w) << S.init_coeffs[k]; }
  std::cout << std::endl;
}
}  // namespace

int main(int argc, char** argv) {
  icccli::Flags F;
  F.str = {{"telemetry_json", ""}, {"output_json", ""}};
  F.num = {{"device", 0.0}};
  F.boolean = {{"verbose", false}};
  try { icccli::parse_flags(argc, argv, F); } catch (const std::exception& e) { std::cerr << "ERROR: " << e.what() << std::endl; return 1; }
  try {
    icccli::Telemetry tel;
    try { tel = icccli::load_telemetry(F.str["telemetry_json"]); } catch (const std::exception& e) { std::cerr << "Could not read: " << F.str["telemetry_json"] << ": " << e.what() << std::endl; return 1; }
    const size_t n = tel.t_ns.size();
    if (tel.acc.size() != 3 * n || tel.gyr.size() != 3 * n) { std::cerr << "Telemetry should have the same amount of timestamps, accelerometer and gyroscope values." << std::endl; return 1; }
    std::vector<double> t(n);
    for (size_t i = 0; i < n; ++i) t[i] = tel.t_ns[i] * 1e-9;
    icc_allan_options o; icc_default_allan_options(&o);
    std::cout << "Loading datastructes\n";
    for (int c = 0; c < 6; ++c) std::cout << kNames[c] << "  num of Cluster " << o.n_clusters << std::endl;
    icc_handle* h = nullptr;
    icc_status st = icc_create(&h, (int)F.num["device"]);
    if (st != ICC_OK) { std::cerr << "icc_create failed (" << st << "): " << icc_last_error(h) << std::endl; return 2; }
    double p[30]; icc_allan_noise z[6]; icc_allan_summary S[6];
    st = icc_allan_variance(h, (int)n, t.data(), tel.acc.data(), tel.gyr.data(), &o, p, z, S);
    if (st != ICC_OK) { std::cerr << "Allan variance failed (" << st << "): " << icc_last_error(h) << std::endl; icc_destroy(h); return 2; }
    const int nf = S[0].n_factors;
    std::vector<int32_t> fac(nf); std::vector<double> tau(nf), s2[6], dev[6];
    for (int c = 0; c < 6; ++c) {
      int32_t len = nf; s2[c].resize(nf); dev[c].resize(nf);
      st = icc_get_allan_curves(h, c, fac.data(), tau.data(), s2[c].data(), dev[c].data(), &len);
      if (st != ICC_OK) { std::cerr << "icc_get_allan_curves failed (" << st << ")" << std::endl; icc_destroy(h); return 2; }
    }
    icc_destroy(h);
    // RunFit (allan_variance_fitter.cc:38-116): the gyroscope channels, then the accelerometer channels
    const double t0 = t.front(), t1 = t.back();
    const char* gyro_title[3] = {"Gyro X ", "Gyro y ", "Gyro z "};
    for (int c = 3; c < 6; ++c) print_calc(kNames[c], (int)n, t0, t1, S[c]);
    for (int c = 3; c < 6; ++c) {
      std::cout << gyro_title[c - 3] << std::endl;
      print_init(S[c]);
      std::cout << " Bias Instability " << z[c].bias_b << " rad/s" << std::endl;
      std::cout << " Bias Instability " << z[c].bias_instability << " rad/s, at " << z[c].bias_instability_tau << " s" << std::endl;
      std::cout << " White Noise " << z[c].white_noise_n << " rad/s" << std::endl;
      std::cout << " White Noise " << z[c].white_noise << " rad/s" << std::endl;
      std::cout << "  bias " << z[c].mean << " degree/s" << std::endl << "-------------------" << std::endl;
    }
    std::cout << "==============================================" << std::endl << "==============================================" << std::endl;
    const char* acc_title[3] = {"acc X ", "acc y ", "acc z "};
    for (int c = 0; c < 3; ++c) print_calc(kNames[c], (int)n, t0, t1, S[c]);
    for (int c = 0; c < 3; ++c) {
      std::cout << acc_title[c] << std::endl;
      print_init(S[c]);
      std::cout << " Bias Instability " << z[c].bias_instability << " m/s^2" << std::endl;
      std::cout << " White Noise " << z[c].white_noise << " m/s^2" << std::endl << "-------------------" << std::endl;
    }
    if (F.boolean["verbose"])
      for (int c = 0; c < 6; ++c)
        std::cout << kNames[c] << ": " << S[c].n_factors << " cluster sizes, " << S[c].n_fit_points << " fitted points, " << S[c].iterations
                  << " dogleg iterations (termination " << S[c].termination << "), cost " << S[c].initial_cost << " -> " << S[c].final_cost << std::endl;
    if (!F.str["output_json"].empty()) {   // the document of io_formats.allan_variance_document
      Value out = Value::object();
      out["n_samples"] = Value((double)n); out["freq"] = Value(S[0].freq); out["period"] = Value(S[0].period);
      out["channels"] = Value::object();
      std::vector<double> facd(fac.begin(), fac.end());
      for (int c = 0; c < 6; ++c) {
        Value ch = Value::object();
        ch["factors"] = array(facd.data(), nf); ch["tau"] = array(tau.data(), nf); ch["sigma2"] = array(s2[c].data(), nf);
        ch["fit_deviation"] = array(dev[c].data(), nf);
        ch["params"] = Value::object();
        for (int k = 0; k < 5; ++k) ch["params"][kParams[k]] = Value(p[5 * c + k]);
        ch["noise"] = Value::object();
        ch["noise"]["mean"] = Value(z[c].mean); ch["noise"]["bias_instability"] = Value(z[c].bias_instability);
        ch["noise"]["bias_instability_tau"] = Value(z[c].bias_instability_tau); ch["noise"]["bias_b"] = Value(z[c].bias_b);
        ch["noise"]["white_noise_n"] = Value(z[c].white_noise_n); ch["noise"]["white_noise"] = Value(z[c].white_noise);
        ch["fit"] = Value::object();
        ch["fit"]["points"] = Value((double)S[c].n_fit_points); ch["fit"]["iterations"] = Value((double)S[c].iterations);
        ch["fit"]["termination"] = Value((double)S[c].termination); ch["fit"]["initial_cost"] = Value(S[c].initial_cost); ch["fit"]["final_cost"] = Value(S[c].final_cost);
        out["channels"][kNames[c]] = ch;
      }
      std::ofstream f(F.str["output_json"]);
      if (!f.is_open()) { std::cerr << "could not write " << F.str["output_json"] << std::endl; return 1; }
      f << iccjson::dump(out, 1) << std::endl;
    }
  } catch (const std::exception& e) { std::cerr << "ERROR: " << e.what() << std::endl; return 1; }
  return 0;
}
