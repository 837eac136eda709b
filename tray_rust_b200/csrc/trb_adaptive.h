// trb_adaptive.h — the Adaptive sampler's schedule and per-pixel decision (src/sampler/adaptive.rs), shared by the host
// (trb_adaptive_schedule, trb_host_adaptive_decide, the round scheduler) and the device (k_adaptive_decide).
//   ad_schedule   Adaptive::new (adaptive.rs:34-49): min / max rounded up to powers of two, step = ((max - min) / 5).next_power_of_two()
//   ad_add        needs_supersampling's average (adaptive.rs:57-67): round 0 an f32 sum, later rounds the cumulative moving average
//                 with the reference's off-by-one, (lum + (i - 1) * avg) / i at the 0-based slot i
//   ad_finish     report_results (adaptive.rs:127-141): stop at samples_taken >= max or when no sample's |lum - avg| / avg > 0.5
// The reference tests every sample of the pixel's list. Correctly rounded subtraction and division are monotone, so the largest
// |lum - avg| / avg over the list is reached at its smallest or its largest luminance: 16 bytes per pixel replace the list.
// fminf / fmaxf skip NaN luminances, and a NaN average (any NaN in the list) makes every comparison false, as in the literal loop.
#pragma once
#include <cstdint>
#include <cmath>
#include "trb_host.h"

namespace trbh {

struct AdSchedule { uint32_t min, max, step, max_per_pixel, rounds; };

// usize::next_power_of_two: 0 -> 1
TRB_HD inline uint32_t ad_pow2(uint32_t v) { uint32_t p = 1; while (p < v) p <<= 1; return p; }

// false: max < min after rounding (the reference's usize subtraction underflows and panics), or beyond 2^24 samples per pixel
TRB_HD inline bool ad_schedule(uint32_t min_in, uint32_t max_in, AdSchedule& s) {
    if (min_in > (1u << 24) || max_in > (1u << 24)) return false;
    s.min = ad_pow2(min_in); s.max = ad_pow2(max_in);
    if (s.max < s.min) return false;
    s.step = ad_pow2((s.max - s.min) / 5u);
    const uint32_t k = (s.max - s.min + s.step - 1u) / s.step; // rounds after the first: samples_taken = min + k * step >= max
    s.rounds = 1u + k;
    s.max_per_pixel = s.min + k * s.step;
    return true;
}
// round r: how many samples, the LD offset (samples_taken after the increment, adaptive.rs:88-101,110,115), the first slot
TRB_HD inline uint32_t ad_count(const AdSchedule& s, uint32_t r) { return r == 0 ? s.min : s.step; }
TRB_HD inline uint32_t ad_offset(const AdSchedule& s, uint32_t r) { return s.min + r * s.step; }
TRB_HD inline uint32_t ad_slot_base(const AdSchedule& s, uint32_t r) { return r == 0 ? 0u : s.min + (r - 1u) * s.step; }

// Colorf::luminance, left to right, never contracted
TRB_HD inline float ad_luminance(float r, float g, float b) { return 0.2126f * r + 0.7152f * g + 0.0722f * b; }

// Per-pixel state: samples taken (bit 31: still sampling), running sum (round 0) or average, smallest and largest luminance.
constexpr uint32_t AD_ACTIVE = 0x80000000u;
struct AdPixel { uint32_t taken; float avg, lmin, lmax; };

TRB_HD inline AdPixel ad_initial() { AdPixel p; p.taken = AD_ACTIVE; p.avg = 0.0f; p.lmin = INFINITY; p.lmax = -INFINITY; return p; }
// one new sample at the 0-based slot `slot` of the pixel's list (round 0: slots 0..min-1, summed in order)
TRB_HD inline void ad_add(AdPixel& p, uint32_t slot, float lum, bool round0) {
    p.lmin = fminf(p.lmin, lum); p.lmax = fmaxf(p.lmax, lum);
    if (round0) p.avg = p.avg + lum;
    else p.avg = (lum + (float)(slot - 1u) * p.avg) / (float)slot;
}
TRB_HD inline bool ad_contrast(float lum, float avg) { return fabsf(lum - avg) / avg > 0.5f; }
// after the round's samples were added: samples_taken, the round-0 average, report_results. Returns whether the pixel goes on.
TRB_HD inline bool ad_finish(AdPixel& p, const AdSchedule& s, uint32_t r) {
    const uint32_t taken = ad_offset(s, r);
    if (r == 0) p.avg = p.avg / (float)s.min; // fold(0.0, +) / samples.len() as f32
    const bool more = taken < s.max && (ad_contrast(p.lmin, p.avg) || ad_contrast(p.lmax, p.avg));
    p.taken = taken | (more ? AD_ACTIVE : 0u);
    return more;
}

} // namespace trbh
