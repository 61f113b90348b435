// kintinuous_b200 -- shared device/host helpers for the sm_90a kernels.
//
// Numerics contract: every kernel in csrc/ is compiled with the reference's own nvcc numerics
// flags (--ftz=true --prec-div=false --prec-sqrt=false, reference CMakeLists.txt:47) and keeps the
// reference's per-element expression order, so that per-pixel / per-voxel results agree with the
// reference's CUDA path bit-for-bit wherever the compiler contracts the same way; reductions use a
// different (fixed, deterministic) summation tree and agree to float rounding.
#pragma once
#include <cuda_runtime.h>
#include <atomic>
#include <stdint.h>
#include <math.h>

namespace kt {

struct Intr { float fx, fy, cx, cy; };
struct Mat33 { float3 r0, r1, r2; };          // row-major rows, same bytes as 9 floats

__host__ __device__ __forceinline__ Intr intr_level(const Intr& k, int level)   // cuda/internal.h:255-259
{
    int div = 1 << level;
    Intr r = {k.fx / div, k.fy / div, k.cx / div, k.cy / div};
    return r;
}

// a.x * b.x + a.y * b.y + a.z * b.z in the contraction nvcc gives the reference's expressions: fma(a.z, b.z, fma(a.x, b.x, a.y * b.y));
// a * b - c * d likewise is fma(a, b, -(c * d)).  Written out so that edits elsewhere cannot flip which product gets fused.
__device__ __forceinline__ float dot3(const float3& a, const float3& b) { return __fmaf_rn(a.z, b.z, __fmaf_rn(a.x, b.x, __fmul_rn(a.y, b.y))); }
__device__ __forceinline__ float3 cross3(const float3& a, const float3& b)
{
    return make_float3(__fmaf_rn(a.y, b.z, -__fmul_rn(a.z, b.y)), __fmaf_rn(a.z, b.x, -__fmul_rn(a.x, b.z)), __fmaf_rn(a.x, b.y, -__fmul_rn(a.y, b.x)));
}
__device__ __forceinline__ float3 sub3(const float3& a, const float3& b) { return make_float3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ float3 add3(const float3& a, const float3& b) { return make_float3(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ float3 scale3(const float3& a, float s) { return make_float3(a.x * s, a.y * s, a.z * s); }
__device__ __forceinline__ float norm3(const float3& a) { return sqrtf(dot3(a, a)); }
__device__ __forceinline__ float3 normalized3(const float3& a) { return scale3(a, rsqrtf(dot3(a, a))); }
__device__ __forceinline__ float3 mul33(const Mat33& m, const float3& v)
{
    return make_float3(dot3(m.r0, v), dot3(m.r1, v), dot3(m.r2, v));
}

__host__ __device__ __forceinline__ int div_up(int a, int b) { return (a + b - 1) / b; }

// Cyclic volume offset reduced to [0, V).  The reference's kernels take the tracker's vWrapCopy -- non-negative but unbounded: it grows by
// `thresh` voxels per +shift (KintinuousTracker.cpp:1075-1085) -- and reduce it with % VOLUME per access (tsdf_volume.cu:612,
// ray_caster.cu:98-110, extract.cu:139).  The kernels here wrap by compare-subtract or mask, so every host wrapper reduces the offset
// once per launch; congruent offsets address the same storage, so results are unchanged.
__host__ __device__ __forceinline__ int wrap_mod(int w, int V) { int r = w % V; return r < 0 ? r + V : r; }
__host__ __device__ __forceinline__ int3 wrap_mod3(const int3& w, int V) { return make_int3(wrap_mod(w.x, V), wrap_mod(w.y, V), wrap_mod(w.z, V)); }

// TSDF fixed point (cuda/device.hpp:67-83, cuda/internal.h:237)
#define KT_DIVISOR 32767
__device__ __forceinline__ short pack_tsdf(float tsdf)
{
    return (short)max(-KT_DIVISOR, min(KT_DIVISOR, __float2int_rz(tsdf * KT_DIVISOR)));
}
__device__ __forceinline__ float unpack_tsdf(short v) { return static_cast<float>(v) / KT_DIVISOR; }

__device__ __forceinline__ float qnan() { return __int_as_float(0x7fffffff); }

} // namespace kt

// error plumbing shared by the host translation units
namespace kt {
void set_error(const char* fmt, ...);
int cuda_check(cudaError_t e, const char* what, const char* file, int line);
// Per-device facts and one-time kernel attribute configuration, cached per device ordinal (kt_config.device lets one process own
// trackers on several GPUs; cudaFuncSetAttribute is per device).
struct DeviceInfo { int sm_count; int smem_optin; unsigned int configured; };
DeviceInfo& device_info();                      // of the CURRENT device
extern std::atomic<long long> g_launches;      // kernels launched by this library (bench.py: gpu_launches); contexts may live on several host threads
}
#define KT_CUDA(expr) do { int _s = kt::cuda_check((expr), #expr, __FILE__, __LINE__); if (_s) return _s; } while (0)
#define KT_LAUNCH_CHECK() do { ++kt::g_launches; int _s = kt::cuda_check(cudaGetLastError(), "kernel launch", __FILE__, __LINE__); if (_s) return _s; } while (0)
