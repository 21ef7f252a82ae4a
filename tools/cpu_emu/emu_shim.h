// DEVELOPMENT AID ONLY -- host stand-ins for the handful of CUDA device intrinsics used by redner_b200/csrc/*.cuh so
// that the per-sample render logic can be compiled with g++ and stepped through / compared against the oracle in a
// container without a GPU.  Nothing under tools/cpu_emu is part of the product: redner_b200/ never loads it and the bench
// never runs it; tests/test_device_code_cpu.py checks this build of the device headers against the golden fixtures.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>
#include <cuda_runtime.h> // vector types + empty __host__/__device__ when compiled by g++
#ifndef __CUDACC__
#define RB_CPU_EMU 1
template <typename T> static inline T __ldg(const T* p) { return *p; }
static inline int __float_as_int(float f) { int i; std::memcpy(&i, &f, 4); return i; }
static inline float __int_as_float(int i) { float f; std::memcpy(&f, &i, 4); return f; }
static inline double __longlong_as_double(long long v) { double d; std::memcpy(&d, &v, 8); return d; }
// CUDA's erfinv (the Gaussian pixel filter's inverse CDF): M. Giles' approximation, refined by Newton steps on std::erf to double
// precision.  |y| < 1 only (the filter scales its argument by erf(3 / sqrt 2)).
static inline double erfinv(double y) {
    double w = -std::log((1.0 - y) * (1.0 + y)), x;
    if (w < 5.0) {
        w -= 2.5;
        double p = 2.81022636e-08;
        p = 3.43273939e-07 + p * w; p = -3.5233877e-06 + p * w; p = -4.39150654e-06 + p * w; p = 0.00021858087 + p * w;
        p = -0.00125372503 + p * w; p = -0.00417768164 + p * w; p = 0.246640727 + p * w; p = 1.50140941 + p * w;
        x = p * y;
    } else {
        w = std::sqrt(w) - 3.0;
        double p = -0.000200214257;
        p = 0.000100950558 + p * w; p = 0.00134934322 + p * w; p = -0.00367342844 + p * w; p = 0.00573950773 + p * w;
        p = -0.0076224613 + p * w; p = 0.00943887047 + p * w; p = 1.00167406 + p * w; p = 2.83297682 + p * w;
        x = p * y;
    }
    for (int i = 0; i < 3; i++) x -= (std::erf(x) - y) / (1.12837916709551257 * std::exp(-x * x));
    return x;
}
#endif
