// Driver of the reference's AllanAcc / AllanGyr (compiled from the reference checkout by the Makefile of this directory).
//   allan_ref <input> <output> <n_clusters> <channels>
// input: int64 n, then n timestamps [s], n x 3 accelerometer [m/s^2], n x 3 gyroscope [rad/s] (float64).  The samples are pushed as
// AllanVarianceFitter's constructor does (pushMPerSec2 / pushRadPerSec); for every channel listed in <channels> (digits 0-5: acc x, y, z,
// gyr x, y, z) calc() runs and the output receives int32 channel, int32 F, then getFactors() (F int32), getTimes() and getVariance()
// (F float64 each).  The reference's console output goes to stdout.
#include "OpenCameraCalibrator/allanvariance/allan_acc.h"
#include "OpenCameraCalibrator/allanvariance/allan_gyr.h"

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

using namespace OpenICC::allanvar;

template <class A>
void write_channel(FILE* o, int c, A& a) {
  a.calc();
  const std::vector<double> tau = a.getTimes(), s2 = a.getVariance();
  const std::vector<int> f = a.getFactors();
  const int32_t F = (int32_t)tau.size();
  std::vector<int32_t> fi(f.begin(), f.begin() + F);
  const int32_t cc = c;
  fwrite(&cc, 4, 1, o); fwrite(&F, 4, 1, o); fwrite(fi.data(), 4, F, o); fwrite(tau.data(), 8, F, o); fwrite(s2.data(), 8, F, o);
}

int main(int argc, char** argv) {
  if (argc != 5) { fprintf(stderr, "usage: allan_ref <input> <output> <n_clusters> <channels>\n"); return 1; }
  FILE* in = fopen(argv[1], "rb");
  if (!in) { perror(argv[1]); return 1; }
  int64_t n = 0;
  if (fread(&n, 8, 1, in) != 1) return 1;
  std::vector<double> t(n), acc(3 * n), gyr(3 * n);
  if (fread(t.data(), 8, n, in) != (size_t)n || fread(acc.data(), 8, 3 * n, in) != (size_t)(3 * n) || fread(gyr.data(), 8, 3 * n, in) != (size_t)(3 * n)) return 1;
  fclose(in);
  const int nc = atoi(argv[3]);
  const std::string channels = argv[4];
  FILE* o = fopen(argv[2], "wb");
  if (!o) { perror(argv[2]); return 1; }
  const char* names[6] = {"acc_x", "acc_y", "acc_z", "gyr_x", "gyr_y", "gyr_z"};
  for (char ch : channels) {
    const int c = ch - '0';
    if (c < 3) {
      AllanAcc a(names[c], nc);
      for (int64_t i = 0; i < n; ++i) a.pushMPerSec2(acc[3 * i + c], t[i]);
      write_channel(o, c, a);
    } else {
      AllanGyr g(names[c], nc);
      for (int64_t i = 0; i < n; ++i) g.pushRadPerSec(gyr[3 * i + c - 3], t[i]);
      write_channel(o, c, g);
    }
  }
  fclose(o);
  return 0;
}
