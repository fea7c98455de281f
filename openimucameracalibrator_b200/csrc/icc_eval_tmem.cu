// Persistent Jacobian evaluation kernel (sm_90a): every warp runs one contiguous run of the packed corner stream (vision items,
// icc_vision_tmem.cuh) or of the packed IMU sample stream (IMU items, icc_imu_tmem.cuh), parking its tensor-core accumulators and
// deferred rows in a lane-private shared-memory park (icc_park.cuh) between the tensor-core and SIMT phases.
//
// One kernel body, TWO launches per evaluation (vision items, then IMU items): the unrolled FP64 recursions make this kernel large,
// and a launch that only walks one phase keeps its instruction working set to that phase.
// Small problems (fewer than a few chunks per warp) stay on the one-warp-per-frame / per-cell kernels of icc_eval.cu, which run
// side by side on two streams and have the shorter single-item latency (launch_eval decides).
//   reference: RSReprojectionCostFunctorSplit<6> / AccelerationCostFunctorSplit<6> / GyroCostFunctorSplit<6>
//   (basalt_spline/ceres_calib_split_residuals.h:319-402, 52-93, 133-169) under Ceres autodiff + LieLocalParameterization.
#include "icc_kernels.h"
#include "icc_vision_tmem.cuh"
#include <cstdlib>
#include "icc_imu_tmem.cuh"

namespace icc {

namespace {

// warps per CTA: per warp a 13.5 KB tile, a 21.3 KB park and its staging slot; six of them fill the 227 KB a block may use on sm_90a
constexpr int EW = 6;
static_assert(tmv::VW == EW && tmi::IW == EW, "one CTA shape");
constexpr size_t SLOT_BYTES = ((sizeof(tmi::ImuSlot) > sizeof(tmv::WarpSlot) ? sizeof(tmi::ImuSlot) : sizeof(tmv::WarpSlot)) + 15) / 16 * 16;
constexpr size_t CONST_BYTES = ((sizeof(VisConst) + sizeof(ImuConst) + 15) / 16) * 16;
constexpr size_t PARK_BYTES = (size_t)PARK_DOUBLES * 32 * sizeof(double);
constexpr size_t SMEM_BYTES = CONST_BYTES + EW * (SLOT_BYTES + PARK_BYTES + (size_t)TILE_COLS * TILE_LD * sizeof(double));
static_assert(SMEM_BYTES <= 227 * 1024, "shared memory of one sm_90a block");

template <int MODEL>
__global__ void __launch_bounds__(EW * 32, 1) eval_tmem_kernel(DeviceProblem P, DeviceState S, double* __restrict__ res_out, int rounds, int groups, int stagger_ns) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  VisConst* KV = reinterpret_cast<VisConst*>(smem_raw);
  ImuConst* KI = reinterpret_cast<ImuConst*>(smem_raw + sizeof(VisConst));
  unsigned char* slots = smem_raw + CONST_BYTES;
  double* tiles = reinterpret_cast<double*>(slots + EW * SLOT_BYTES);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double* tile = tiles + warp * (TILE_COLS * TILE_LD);
  double* ta = tiles + EW * (TILE_COLS * TILE_LD) + warp * (PARK_DOUBLES * 32) + lane;   // this lane's column of the warp's park

  tmv::init_const(KV, P, S, MODEL);
  tmi::init_const(KI, P, S);
  for (int i = lane; i < TILE_COLS * TILE_LD; i += 32) tile[i] = 0.0;
  __syncthreads();
  NeLayout L; L.ne = P.ne; L.off_E = P.ne_off_E; L.off_C = P.ne_off_C; L.off_g = P.ne_off_g; L.off_cost = P.ne_off_cost; L.nk = P.nk; L.nb = P.nb; L.ldb = P.ldb;

  const int gw = warp * gridDim.x + blockIdx.x;           // global warp: consecutive runs land on different SMs
  // lockstep groups: the whole CTA (groups == 1) or `groups` equal sets of warps (warp % groups; groups divides EW), each with its
  // own named barriers and started `stagger_ns` apart, so that one group's tensor-core phase meets the others' SIMT phases
  const int grp = warp % groups, bar_id = 1 + grp, bar_n = EW * 32 / groups;
  if (groups > 1 && stagger_ns > 0) for (int g = 0; g < grp; ++g) __nanosleep(stagger_ns);
  if (P.n_vitems > 0) {
    if (gw < P.n_vitems) tmv::run_item<MODEL>(P, S, KV, reinterpret_cast<tmv::WarpSlot*>(slots + warp * SLOT_BYTES), tile, ta, L, P.vitems[gw], res_out, lane, rounds, bar_id, bar_n);
    else for (int r = 0; r < rounds; ++r) asm volatile("bar.sync %0, %1;" :: "r"(bar_id), "r"(bar_n) : "memory");
  } else if (P.n_iitems > 0) {           // (a launch carries one item type: launch_eval_tmem)
    if (gw < P.n_iitems) tmi::run_item(P, S, KI, reinterpret_cast<tmi::ImuSlot*>(slots + warp * SLOT_BYTES), tile, ta, L, P.iitems[gw], res_out, lane, rounds, bar_id, bar_n);
    else for (int r = 0; r < rounds; ++r) { asm volatile("bar.sync %0, %1;" :: "r"(bar_id), "r"(bar_n) : "memory"); asm volatile("bar.sync %0, %1;" :: "r"(bar_id + 6), "r"(bar_n) : "memory"); }
  }
}

template <int MODEL>
int launch_model(const DeviceProblem& P, const DeviceState& S, double* residuals_out, int grid, size_t smem, cudaStream_t st) {
  static bool attr_done = false;
  if (!attr_done) {
    if (cudaFuncSetAttribute(eval_tmem_kernel<MODEL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return 1;
    attr_done = true;
  }
  // loose lockstep: warps start every chunk together (one named barrier per chunk), so that they walk the same unrolled code at the
  // same time (instruction-cache locality).  The whole CTA steps together by default (ICC_TMEM_GROUPS = 2, 3 or 6 splits it into
  // that many groups, ICC_TMEM_STAGGER_NS delays group g by g x ns, ICC_TMEM_NO_LOCKSTEP lets every warp run free).
  const int rounds = getenv("ICC_TMEM_NO_LOCKSTEP") ? 0 : P.n_vitems > 0 ? (P.n_vchunks + P.n_vitems - 1) / P.n_vitems : P.n_iitems > 0 ? (P.n_ichunks + P.n_iitems - 1) / P.n_iitems : 0;
  const char* eg = getenv("ICC_TMEM_GROUPS"); const char* es = getenv("ICC_TMEM_STAGGER_NS");
  const int gq = eg ? atoi(eg) : 1, groups = (gq == 2 || gq == 3 || gq == 6) ? gq : 1, stagger_ns = es ? atoi(es) : 0;
  static_assert(EW % 2 == 0 && EW % 3 == 0, "lockstep groups divide the CTA");
  eval_tmem_kernel<MODEL><<<grid, EW * 32, smem, st>>>(P, S, residuals_out, rounds, groups, stagger_ns);
  return 0;
}

}  // namespace

int eval_tmem_warps() { return EW; }

// P.vitems[k] / P.iitems[k] is the run of global warp k (icc_api.cu cuts each stream into at most sm_count * eval_tmem_warps() runs);
// vision and IMU items go out as separate launches of the same kernel.
int launch_eval_tmem(const DeviceProblem& P, const DeviceState& S, double* residuals_out, int sm_count, cudaStream_t st) {
  const size_t smem = SMEM_BYTES;
  for (int pass = 0; pass < 2; ++pass) {
    DeviceProblem Q = P;
    if (pass == 0) Q.n_iitems = 0; else Q.n_vitems = 0;
    const int n = pass == 0 ? Q.n_vitems : Q.n_iitems;
    if (n <= 0) continue;
    const int grid = (n + EW - 1) / EW < sm_count ? (n + EW - 1) / EW : sm_count;
    int e = 1;
    switch (P.model) {   // one instantiation per camera model: only that model's projection code is resident in the instruction cache
      case CAM_PINHOLE: e = launch_model<CAM_PINHOLE>(Q, S, residuals_out, grid, smem, st); break;
      case CAM_PINHOLE_RADTAN: e = launch_model<CAM_PINHOLE_RADTAN>(Q, S, residuals_out, grid, smem, st); break;
      case CAM_FISHEYE: e = launch_model<CAM_FISHEYE>(Q, S, residuals_out, grid, smem, st); break;
      case CAM_FOV: e = launch_model<CAM_FOV>(Q, S, residuals_out, grid, smem, st); break;
      case CAM_DIVISION_UNDISTORTION: e = launch_model<CAM_DIVISION_UNDISTORTION>(Q, S, residuals_out, grid, smem, st); break;
      case CAM_DOUBLE_SPHERE: e = launch_model<CAM_DOUBLE_SPHERE>(Q, S, residuals_out, grid, smem, st); break;
      case CAM_EXTENDED_UNIFIED: e = launch_model<CAM_EXTENDED_UNIFIED>(Q, S, residuals_out, grid, smem, st); break;
      default: return 1;
    }
    if (e) return 1;
    count_launch();
  }
  return cudaGetLastError() == cudaSuccess ? 0 : 1;
}

}  // namespace icc
