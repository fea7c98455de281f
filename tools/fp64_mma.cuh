// The FP64 tensor-core shapes of mma.sync that the microbenchmarks time: m8n8k4 (sm_80 on), and the m16n8k4 / m16n8k8 /
// m16n8k16 shapes sm_90 added.
#pragma once

enum Shape { M8N8K4, M16N8K4, M16N8K8, M16N8K16 };

// One warp-wide FP64 MMA of the given shape on one accumulator fragment (ACC doubles per lane); every A and B operand
// register holds the same value, which does not change the instruction's cost.
template <Shape S> struct Mma;
template <> struct Mma<M8N8K4> {
  static constexpr int ACC = 2; static constexpr double FLOP = 8 * 8 * 4 * 2; static constexpr const char* name = "m8n8k4";
  static __device__ __forceinline__ void run(double* d, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(d[0]), "+d"(d[1]) : "d"(a), "d"(b));
  }
};
template <> struct Mma<M16N8K4> {
  static constexpr int ACC = 4; static constexpr double FLOP = 16 * 8 * 4 * 2; static constexpr const char* name = "m16n8k4";
  static __device__ __forceinline__ void run(double* d, double a, double b) {
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                 : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3]) : "d"(a), "d"(a), "d"(b));
  }
};
template <> struct Mma<M16N8K8> {
  static constexpr int ACC = 4; static constexpr double FLOP = 16 * 8 * 8 * 2; static constexpr const char* name = "m16n8k8";
  static __device__ __forceinline__ void run(double* d, double a, double b) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3]) : "d"(a), "d"(a), "d"(a), "d"(a), "d"(b), "d"(b));
  }
};
template <> struct Mma<M16N8K16> {
  static constexpr int ACC = 4; static constexpr double FLOP = 16 * 8 * 16 * 2; static constexpr const char* name = "m16n8k16";
  static __device__ __forceinline__ void run(double* d, double a, double b) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, {%0,%1,%2,%3};"
                 : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
                 : "d"(a), "d"(a), "d"(a), "d"(a), "d"(a), "d"(a), "d"(a), "d"(a), "d"(b), "d"(b), "d"(b), "d"(b));
  }
};

