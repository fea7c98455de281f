// Persistent Jacobian evaluation kernel (sm_90a): every warp runs one contiguous run of the packed corner stream (vision items,
// icc_vision_tmem.cuh) or of the packed IMU sample stream (IMU items, icc_imu_tmem.cuh), with its tensor-core accumulators in
// registers and its deferred rows parked in a lane-private shared-memory park (icc_park.cuh) between the SIMT and tensor-core phases.
//
// TWO launches per evaluation (vision items, then IMU items), each an instantiation with its own CTA shape: the unrolled FP64
// recursions make this kernel large, and a launch that only walks one item type keeps its instruction working set to that type.
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

constexpr int IMU_ITEMS = -1;          // the MODEL argument of the IMU-item instantiation (IMU items do not depend on the camera model)

// One thread per SO(3) knot increment: the table the item kernels stage their windows from.  Each increment's log and Jr^-1 are formed
// once per evaluation, with every lane busy, instead of once per staged window on five lanes of a warp its CTA's barrier waits for.
// The vision launch behind it may start at once (programmatic dependent launch): its CTAs take the SMs this grid leaves free, set up
// their shared memory and wait for the table at griddepcontrol.wait.
__global__ void __launch_bounds__(128) incr_table_kernel(const double4* __restrict__ so3, int n, double* __restrict__ tab) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) incr_table_entry(so3, i, n, tab);
}

// CTA shape per item type: per warp a 13.5 KB tile, a lane-private park and a staging slot, plus the item type's constants.
//   vision items: 8 warps x (13.5 KB tile + 9 KB park of the y row + 2.1 KB slot);
//   IMU items:    8 warps x (13.5 KB tile + 10.8 KB park of the deferred rows 1 and 2 + 2.6 KB slot).
template <int MODEL>
struct Cta {
  static constexpr bool imu = MODEL == IMU_ITEMS;
  static constexpr int warps = imu ? tmi::IW : tmv::VW;
  static constexpr size_t const_bytes = ((imu ? sizeof(ImuConst) : sizeof(VisConst)) + 15) / 16 * 16;
  static constexpr size_t slot_bytes = ((imu ? sizeof(tmi::ImuSlot) : sizeof(tmv::WarpSlot)) + 15) / 16 * 16;
  static constexpr int park_doubles = imu ? tmi::PARK_N : tmv::PARK_N;
  static constexpr size_t smem_bytes = const_bytes + warps * (slot_bytes + (size_t)park_doubles * 32 * sizeof(double) + (size_t)TILE_COLS * TILE_LD * sizeof(double));
  static_assert(smem_bytes <= 227 * 1024, "shared memory of one sm_90a block");
};

// MODEL >= 0: vision items of that camera model (one instantiation per model: only that model's projection code is resident in the
// instruction cache); VIS_TANGENT: vision items of the tangent reprojection error, whatever the model; IMU_ITEMS: IMU items.
template <int MODEL>
__global__ void __launch_bounds__(Cta<MODEL>::warps * 32, 1) eval_tmem_kernel(DeviceProblem P, DeviceState S, double* __restrict__ res_out, int rounds, int groups, int stagger_ns, TangentMeas T) {
  using C = Cta<MODEL>;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned char* slots = smem_raw + C::const_bytes;
  double* tiles = reinterpret_cast<double*>(slots + C::warps * C::slot_bytes);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double* tile = tiles + warp * (TILE_COLS * TILE_LD);
  double* ta = tiles + C::warps * (TILE_COLS * TILE_LD) + warp * (C::park_doubles * 32) + lane;   // this lane's column of the warp's park

  if constexpr (C::imu) tmi::init_const(reinterpret_cast<ImuConst*>(smem_raw), P, S);
  else tmv::init_const(reinterpret_cast<VisConst*>(smem_raw), P, S, MODEL);
  for (int i = lane; i < TILE_COLS * TILE_LD; i += 32) tile[i] = 0.0;
  __syncthreads();
  // Programmatic dependent launch (launch_eval_tmem): the vision items wait here for the increment table of the launch before them, then
  // let the IMU launch go, whose CTAs take each SM as the vision CTA there retires.  The IMU items need nothing the vision items write
  // (both only add into the normal equations) and the table was complete before the vision items passed this point, so they wait for
  // the vision grid only at their end: whatever follows the IMU launch in the stream then follows both.
  if constexpr (!C::imu) {
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  }
  NeLayout L; L.ne = P.ne; L.off_E = P.ne_off_E; L.off_C = P.ne_off_C; L.off_g = P.ne_off_g; L.off_cost = P.ne_off_cost; L.nk = P.nk; L.nb = P.nb; L.ldb = P.ldb;

  const int gw = warp * gridDim.x + blockIdx.x;           // global warp: consecutive runs land on different SMs
  // lockstep groups: the whole CTA (groups == 1) or `groups` equal sets of warps (warp % groups; groups divides the CTA's warps), each
  // with its own named barrier (id 1 + group) and started `stagger_ns` apart, so that one group's tensor-core phase meets the others'
  // SIMT phases
  static_assert(C::warps < 16, "one named barrier per lockstep group, ids 1..groups");
  const int grp = warp % groups, bar_id = 1 + grp, bar_n = C::warps * 32 / groups;
  if (groups > 1 && stagger_ns > 0) for (int g = 0; g < grp; ++g) __nanosleep(stagger_ns);
  if constexpr (C::imu) {
    if (gw < P.n_iitems) tmi::run_item(P, S, reinterpret_cast<const ImuConst*>(smem_raw), reinterpret_cast<tmi::ImuSlot*>(slots + warp * C::slot_bytes), tile, ta, L, P.iitems[gw], res_out, lane, rounds, bar_id, bar_n);
    else for (int r = 0; r < rounds; ++r) { asm volatile("bar.sync %0, %1;" :: "r"(bar_id), "r"(bar_n) : "memory"); asm volatile("bar.sync %0, %1;" :: "r"(bar_id), "r"(bar_n) : "memory"); }
    asm volatile("griddepcontrol.wait;" ::: "memory");   // returns at once unless launched behind the vision items
  } else {
    if (gw < P.n_vitems) tmv::run_item<MODEL>(P, T, S, reinterpret_cast<const VisConst*>(smem_raw), reinterpret_cast<tmv::WarpSlot*>(slots + warp * C::slot_bytes), tile, ta, L, P.vitems[gw], res_out, lane, rounds, bar_id, bar_n);
    else for (int r = 0; r < rounds; ++r) asm volatile("bar.sync %0, %1;" :: "r"(bar_id), "r"(bar_n) : "memory");
  }
}

// n_items: the launch's runs (P.n_vitems or P.n_iitems), n_chunks: the chunks of its stream; early: programmatic dependent launch on the
// kernel before it in the stream (the increment table for the vision items, the vision items for the IMU items)
template <int MODEL>
int launch_model(const DeviceProblem& P, const DeviceState& S, double* residuals_out, int n_items, int n_chunks, int sm_count, cudaStream_t st, TangentMeas T, bool early) {
  using C = Cta<MODEL>;
  static bool attr_done = false;
  if (!attr_done) {
    if (cudaFuncSetAttribute(eval_tmem_kernel<MODEL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::smem_bytes) != cudaSuccess) return 1;
    attr_done = true;
  }
  const int grid = (n_items + C::warps - 1) / C::warps < sm_count ? (n_items + C::warps - 1) / C::warps : sm_count;
  // Every warp runs free by default.  Loose lockstep -- warps start every chunk together at a named barrier, so that they walk the same
  // unrolled code at the same time (instruction-cache locality) -- is opt-in: ICC_TMEM_GROUPS = g steps g groups of warps (1: the whole
  // CTA; any g that divides the CTA's warps: 2, 4 or 8 for both item types, each group on its own named barrier), ICC_TMEM_STAGGER_NS
  // delays group g by g x ns, ICC_TMEM_NO_LOCKSTEP overrides both.  Since windows are copied from the increment table, the barrier
  // costs more than it saves: on config 4 the whole-CTA lockstep made the vision launch 168 us instead of 158 us (DESIGN 3.1).
  const char* eg = getenv("ICC_TMEM_GROUPS"); const char* es = getenv("ICC_TMEM_STAGGER_NS");
  const int rounds = eg && !getenv("ICC_TMEM_NO_LOCKSTEP") ? (n_chunks + n_items - 1) / n_items : 0;
  const int gq = eg ? atoi(eg) : 1, groups = (gq > 1 && gq <= C::warps && C::warps % gq == 0) ? gq : 1, stagger_ns = es ? atoi(es) : 0;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(C::warps * 32); cfg.dynamicSmemBytes = C::smem_bytes; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = early ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, eval_tmem_kernel<MODEL>, P, S, residuals_out, rounds, groups, stagger_ns, T) == cudaSuccess ? 0 : 1;
}

}  // namespace

int eval_tmem_warps(bool imu_items) { return imu_items ? Cta<IMU_ITEMS>::warps : Cta<0>::warps; }

// P.vitems[k] / P.iitems[k] is the run of global warp k (icc_api.cu cuts each stream into at most sm_count * eval_tmem_warps(type) runs);
// the increment table of S first, then vision and IMU items as separate launches, each with its own CTA shape.
int launch_eval_tmem(const DeviceProblem& P, const DeviceState& S, double* residuals_out, int sm_count, cudaStream_t st, const TangentMeas* tan) {
  const TangentMeas T = tan ? *tan : TangentMeas{nullptr, nullptr, 0.0};
  if (P.n_vitems <= 0 && P.n_iitems <= 0) return 0;
  if (!P.incr || P.n_so3 < SPLINE_N) return 1;
  {                                    // the increment table of the state evaluated here (S), never one left by another state
    const int n = P.n_so3 - 1;
    incr_table_kernel<<<(n + 127) / 128, 128, 0, st>>>(S.so3, n, P.incr);
    count_launch();
  }
  if (P.n_vitems > 0) {
    DeviceProblem Q = P;
    Q.n_iitems = 0;
    const int nv = P.n_vitems, nc = P.n_vchunks;
    int e = 1;
    if (tan) e = launch_model<VIS_TANGENT>(Q, S, residuals_out, nv, nc, sm_count, st, T, true);
    else switch (P.model) {
      case CAM_PINHOLE: e = launch_model<CAM_PINHOLE>(Q, S, residuals_out, nv, nc, sm_count, st, T, true); break;
      case CAM_PINHOLE_RADTAN: e = launch_model<CAM_PINHOLE_RADTAN>(Q, S, residuals_out, nv, nc, sm_count, st, T, true); break;
      case CAM_FISHEYE: e = launch_model<CAM_FISHEYE>(Q, S, residuals_out, nv, nc, sm_count, st, T, true); break;
      case CAM_FOV: e = launch_model<CAM_FOV>(Q, S, residuals_out, nv, nc, sm_count, st, T, true); break;
      case CAM_DIVISION_UNDISTORTION: e = launch_model<CAM_DIVISION_UNDISTORTION>(Q, S, residuals_out, nv, nc, sm_count, st, T, true); break;
      case CAM_DOUBLE_SPHERE: e = launch_model<CAM_DOUBLE_SPHERE>(Q, S, residuals_out, nv, nc, sm_count, st, T, true); break;
      case CAM_EXTENDED_UNIFIED: e = launch_model<CAM_EXTENDED_UNIFIED>(Q, S, residuals_out, nv, nc, sm_count, st, T, true); break;
      case CAM_OMNI_RADTAN: e = launch_model<CAM_OMNI_RADTAN>(Q, S, residuals_out, nv, nc, sm_count, st, T, true); break;
      case CAM_SCARAMUZZA: e = launch_model<CAM_SCARAMUZZA>(Q, S, residuals_out, nv, nc, sm_count, st, T, true); break;
      case CAM_PINHOLE_RATIONAL: e = launch_model<CAM_PINHOLE_RATIONAL>(Q, S, residuals_out, nv, nc, sm_count, st, T, true); break;
      case CAM_FISHEYE_RADTAN: e = launch_model<CAM_FISHEYE_RADTAN>(Q, S, residuals_out, nv, nc, sm_count, st, T, true); break;
      default: return 1;
    }
    if (e) return 1;
    count_launch();
  }
  if (P.n_iitems > 0) {
    DeviceProblem Q = P;
    Q.n_vitems = 0;
    if (launch_model<IMU_ITEMS>(Q, S, residuals_out, P.n_iitems, P.n_ichunks, sm_count, st, T, P.n_vitems > 0)) return 1;
    count_launch();
  }
  return cudaGetLastError() == cudaSuccess ? 0 : 1;
}

}  // namespace icc
