/* A plain-C caller of trb_illumination (include/trb.h): it compiles and links against libtrb with nothing but the header, pins
 * the layout of trb_illum_ray, prints every sizeof / offsetof, and prints the status of each entry point called with null or
 * out-of-range arguments (checked before any device is touched, so it runs without a GPU). */
#include <stddef.h>
#include <stdio.h>
#include "trb.h"

_Static_assert(sizeof(trb_illum_ray) == 48, "trb_illum_ray is 48 bytes");
_Static_assert(offsetof(trb_illum_ray, min_t) == 24 && offsetof(trb_illum_ray, time) == 32 && offsetof(trb_illum_ray, key) == 36 &&
               offsetof(trb_illum_ray, sample) == 40, "trb_illum_ray layout");
_Static_assert(TRB_QUERY_CLAMP == 32u, "TRB_QUERY_CLAMP");

#define F(T, f) printf(#T "." #f " %d\n", (int)offsetof(T, f))

int main(void) {
    printf("trb_illum_ray sizeof %d\n", (int)sizeof(trb_illum_ray));
    F(trb_illum_ray, o); F(trb_illum_ray, d); F(trb_illum_ray, min_t); F(trb_illum_ray, max_t); F(trb_illum_ray, time);
    F(trb_illum_ray, key); F(trb_illum_ray, sample); F(trb_illum_ray, pad);
    trb_illum_ray ray = {{0, 0, 0}, {0, 0, 1}, 0.0f, 1.0f, 0.0f, 7u, 0u, 0u};
    float rgb[3];
    trb_stats st;
    printf("status trb_illumination %d\n", (int)trb_illumination(NULL, 1, &ray, 1, 1, rgb, TRB_QUERY_CLAMP, &st));
    printf("status trb_illumination_device %d\n", (int)trb_illumination_device(NULL, 1, &ray, 1, 1, rgb, 0, NULL, NULL));
    printf("status trb_illumination_spp0 %d\n", (int)trb_illumination(NULL, 1, &ray, 0, 1, rgb, 0, &st));
    printf("status TRB_INVALID_ARG %d\n", (int)TRB_INVALID_ARG);
    return 0;
}
