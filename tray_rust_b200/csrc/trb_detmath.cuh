// trb_detmath.cuh — device implementation of the "detmath" contract (DESIGN.md, "Determinism
// contract"): a fixed sequence of IEEE-754 binary32 operations for sin/cos/acos/atan2/exp/log/pow
// and the counter-based RNG + index permutation that replace rand::StdRng in the reference
// (/root/reference/src/exec/multithreaded.rs:79, src/sampler/ld.rs:55-63, src/integrator/path.rs:99).
//
// The reference calls the platform libm (Rust f32::sin etc.: src/mc.rs:50, src/bxdf/microfacet/
// beckmann.rs:35-46, src/bxdf/merl.rs:62-75); libdevice and glibc differ in the last ulp, so this
// translation unit is compiled with --fmad=false and evaluates these fixed polynomial sequences
// (Cephes single-precision kernels) instead, which makes every camera sample reproducible on any
// IEEE machine. Written for sm_90a; nothing here is shared with oracle/. The TRB_DM functions compile for the host as well,
// with the same operations, so host code that calls them (trb_host_film_to_srgb8) gets the device's bits.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>
#include <cuda_runtime.h>

namespace trb {

#define TRB_PI 3.14159265358979323846f
#define TRB_PIO2 1.57079632679489661923f
#define TRB_PIO4 0.78539816339744830962f
#define TRB_INV_PI 0.318309886183790671f
#define TRB_EPS 1.1920929e-7f

#define TRB_DM __host__ __device__ __forceinline__
TRB_DM float bits_f32(uint32_t u) {
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float f; memcpy(&f, &u, 4); return f;
#endif
}
TRB_DM uint32_t f32_bits(float f) {
#ifdef __CUDA_ARCH__
    return __float_as_uint(f);
#else
    uint32_t u; memcpy(&u, &f, 4); return u;
#endif
}
TRB_DM float pow2i(int k) { return bits_f32((uint32_t)(k + 127) << 23); }

// Cody-Waite reduction to [-pi/4, pi/4]; quadrant in q. |x| <= 1e5.
TRB_DM float reduce_pio2(float x, int& q) {
    float kf = rintf(x * 0.636619772367581343f);
    q = (int)kf;
    float r = x - kf * 1.5703125f;
    r = r - kf * 4.837512969970703125e-4f;
    r = r - kf * 7.54978995489188216e-8f;
    return r;
}
TRB_DM float sin_kernel(float r) {
    float z = r * r;
    return r + r * z * (-1.6666654611e-1f + z * (8.3321608736e-3f + z * -1.9515295891e-4f));
}
TRB_DM float cos_kernel(float r) {
    float z = r * r;
    return 1.0f - 0.5f * z + z * z * (4.166664568298827e-2f + z * (-1.388731625493765e-3f + z * 2.443315711809948e-5f));
}
// sin and cos of the same angle share the reduction
TRB_DM void dsincos(float x, float& s, float& c) {
    if (!(fabsf(x) <= 1.0e5f)) { s = x - x; c = x - x; return; }
    int q;
    float r = reduce_pio2(x, q);
    float sk = sin_kernel(r), ck = cos_kernel(r);
    switch (q & 3) {
        case 0: s = sk; c = ck; break;
        case 1: s = ck; c = -sk; break;
        case 2: s = -sk; c = -ck; break;
        default: s = -ck; c = sk; break;
    }
}
TRB_DM float dsin(float x) { float s, c; dsincos(x, s, c); return s; }
TRB_DM float dcos(float x) { float s, c; dsincos(x, s, c); return c; }

TRB_DM float asin_kernel(float z) {
    float z2 = z * z;
    float p = ((((4.2163199048e-2f * z2 + 2.4181311049e-2f) * z2 + 4.5470025998e-2f) * z2 + 7.4953002686e-2f) * z2 + 1.6666752422e-1f);
    return z + z * z2 * p;
}
TRB_DM float dacos(float x) {
    if (x != x) return x;
    if (x >= 1.0f) return 0.0f;
    if (x <= -1.0f) return TRB_PI;
    if (x > 0.5f) return 2.0f * asin_kernel(sqrtf(0.5f * (1.0f - x)));
    if (x < -0.5f) return TRB_PI - 2.0f * asin_kernel(sqrtf(0.5f * (1.0f + x)));
    return TRB_PIO2 - asin_kernel(x);
}
__device__ __forceinline__ float atan_pos(float t) {
    float y0, u;
    if (t > 2.414213562373095f) { y0 = TRB_PIO2; u = -(1.0f / t); }
    else if (t > 0.4142135623730950f) { y0 = TRB_PIO4; u = (t - 1.0f) / (t + 1.0f); }
    else { y0 = 0.0f; u = t; }
    float z = u * u;
    float p = (((8.05374449538e-2f * z - 1.38776856032e-1f) * z + 1.99777106478e-1f) * z - 3.33329491539e-1f) * z * u + u;
    return y0 + p;
}
__device__ __forceinline__ float datan2(float y, float x) {
    if (x != x || y != y) return x + y;
    float ax = fabsf(x), ay = fabsf(y);
    float a;
    if (ax == 0.0f && ay == 0.0f) a = 0.0f;
    else if (ax == __int_as_float(0x7f800000) && ay == __int_as_float(0x7f800000)) a = TRB_PIO4;
    else a = atan_pos(ay / ax);
    if (x < 0.0f) a = TRB_PI - a;
    return y < 0.0f ? -a : a;
}
TRB_DM float dexp(float x) {
    if (x != x) return x;
    if (x > 88.72283905206835f) return bits_f32(0x7f800000u);
    if (x < -87.33654475055310f) return 0.0f;
    float kf = floorf(1.44269504088896341f * x + 0.5f);
    float r = x - kf * 0.693359375f;
    r = r - kf * -2.12194440e-4f;
    float z = r * r;
    float p = (((((1.9875691500e-4f * r + 1.3981999507e-3f) * r + 8.3334519073e-3f) * r + 4.1665795894e-2f) * r + 1.6666665459e-1f) * r + 5.0000001201e-1f) * z + r + 1.0f;
    int k = (int)kf;
    if (k > 127) { p = p * 2.0f; k -= 1; }
    return p * pow2i(k);
}
TRB_DM float dlog(float x) {
    if (x != x) return x;
    if (x < 0.0f) return x - x + bits_f32(0x7fc00000u);
    if (x == 0.0f) return bits_f32(0xff800000u);
    if (x == bits_f32(0x7f800000u)) return x;
    int e = 0;
    if (x < 1.17549435e-38f) { x = x * 8388608.0f; e = -23; }
    uint32_t b = f32_bits(x);
    e += (int)((b >> 23) & 0xffu) - 126;
    float m = bits_f32((b & 0x007fffffu) | 0x3f000000u);
    if (m < 0.707106781186547524f) { e -= 1; m = m + m - 1.0f; }
    else { m = m - 1.0f; }
    float z = m * m;
    float y = ((((((((7.0376836292e-2f * m - 1.1514610310e-1f) * m + 1.1676998740e-1f) * m - 1.2420140846e-1f) * m + 1.4249322787e-1f) * m - 1.6668057665e-1f) * m + 2.0000714765e-1f) * m - 2.4999993993e-1f) * m + 3.3333331174e-1f) * m * z;
    float fe = (float)e;
    y = y + -2.12194440e-4f * fe;
    y = y + -0.5f * z;
    z = m + y;
    z = z + 0.693359375f * fe;
    return z;
}
TRB_DM float dpow(float x, float y) { return dexp(y * dlog(x)); }

// ---- counter RNG ---------------------------------------------------------------------
__host__ __device__ __forceinline__ uint32_t mix32(uint32_t x) {
    x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
    return x;
}
// partial hash states let a thread hoist the (seed, pixel) and (seed, pixel, sample) prefixes
__host__ __device__ __forceinline__ uint32_t rng_seed(uint32_t seed) { return mix32(seed ^ 0x9e3779b9U); }
__host__ __device__ __forceinline__ uint32_t rng_absorb(uint32_t h, uint32_t v) { return mix32(h ^ v); }
__host__ __device__ __forceinline__ uint32_t scramble_of(uint32_t h) { return h == 0xffffffffU ? 0xfffffffeU : h; }
__host__ __device__ __forceinline__ float unit_f32(uint32_t h) { return (float)(h >> 8) * (1.0f / 16777216.0f); }

__host__ __device__ __forceinline__ uint32_t permute_index(uint32_t i, uint32_t l, uint32_t p) {
    uint32_t w = l - 1;
    w |= w >> 1; w |= w >> 2; w |= w >> 4; w |= w >> 8; w |= w >> 16;
    do {
        i ^= p; i *= 0xe170893dU;
        i ^= p >> 16;
        i ^= (i & w) >> 4;
        i ^= p >> 8; i *= 0x0929eb3fU;
        i ^= p >> 23;
        i ^= (i & w) >> 1; i *= 1 | p >> 27;
        i *= 0x6935fa69U;
        i ^= (i & w) >> 11; i *= 0x74dcb303U;
        i ^= (i & w) >> 2; i *= 0x9e501cc3U;
        i ^= (i & w) >> 2; i *= 0xc860a3dfU;
        i &= w;
        i ^= i >> 5;
    } while (i >= l);
    i += p % l; /* rotation by the key without 32-bit wrap-around (i, p % l < l) */
    return i >= l ? i - l : i;
}

// stream addressing (DESIGN.md "RNG")
constexpr uint32_t PIXEL_STREAM = 0xffffffffU;
constexpr uint32_t AD_PIXEL_STREAM0 = 0xfffffffeU; // Adaptive sampler, round r: AD_PIXEL_STREAM0 - r (camera-sample slots stay below 2^25)
enum { PX_POS0 = 0, PX_POS1 = 1, PX_POS_PERM = 2, PX_TIME = 3, PX_TIME_PERM = 4 };
enum { S_L0 = 0, S_L1 = 1, S_L_PERM = 2, S_B0 = 3, S_B1 = 4, S_B_PERM = 5, S_P0 = 6, S_P1 = 7, S_P_PERM = 8,
       S_LC = 9, S_LC_PERM = 10, S_BC = 11, S_BC_PERM = 12, S_PC = 13, S_PC_PERM = 14, S_RR = 32 };

// sampler::ld::{van_der_corput, sobol} (src/sampler/ld.rs:95-119)
__host__ __device__ __forceinline__ float ld_vdc(uint32_t n, uint32_t scramble) {
#ifdef __CUDA_ARCH__
    n = __brev(n);
#else
    n = (n << 16) | (n >> 16);
    n = ((n & 0x00ff00ffu) << 8) | ((n & 0xff00ff00u) >> 8);
    n = ((n & 0x0f0f0f0fu) << 4) | ((n & 0xf0f0f0f0u) >> 4);
    n = ((n & 0x33333333u) << 2) | ((n & 0xccccccccu) >> 2);
    n = ((n & 0x55555555u) << 1) | ((n & 0xaaaaaaaau) >> 1);
#endif
    n ^= scramble;
    return fminf((float)((n >> 8) & 0xffffffu) / 16777216.0f, 1.0f - TRB_EPS);
}
__host__ __device__ __forceinline__ float ld_sobol(uint32_t n, uint32_t scramble) {
    uint32_t i = 1u << 31;
    while (n != 0) {
        if (n & 1u) scramble ^= i;
        n >>= 1;
        i ^= i >> 1;
    }
    return fminf((float)((scramble >> 8) & 0xffffffu) / 16777216.0f, 1.0f - TRB_EPS);
}

// Rust `f as usize` into 32 bits: truncation toward zero, saturating, NaN -> 0
TRB_DM uint32_t f2u(float f) {
#ifdef __CUDA_ARCH__
    return __float2uint_rz(f);
#else
    return f != f || f <= 0.0f ? 0u : (f >= 4294967296.0f ? 0xffffffffu : (uint32_t)f);
#endif
}

// One pixel of RenderTarget::get_render (render_target.rs:185-210) and of the master's Image::get_srgb8 (film/image.rs:53-67),
// with Colorf::clamp and Colorf::to_srgb (color.rs:36-72): rgb / weight, clamped to [0, 1], sRGB, then (c * 255) as u8. A pixel
// whose weight is not > 0 stays black. k_srgb8 (trb_film_to_srgb8) and trb_host_film_to_srgb8 both call this, so the device and
// the host convert a film to the same bytes.
TRB_DM void srgb8_pixel(float r, float g, float b, float w, uint8_t* o) {
    o[0] = 0; o[1] = 0; o[2] = 0;
    if (w > 0.0f) {
        const float v[3] = {r / w, g / w, b / w};
        for (int k = 0; k < 3; ++k) {
            const float x = v[k] < 0.0f ? 0.0f : (v[k] > 1.0f ? 1.0f : v[k]);
            const float s = x <= 0.0031308f ? 12.92f * x : (1.0f + 0.055f) * dpow(x, 1.0f / 2.4f) - 0.055f;
            const float q = s * 255.0f;
            o[k] = (uint8_t)f2u(q > 255.0f ? 255.0f : q);
        }
    }
}

} // namespace trb
