/* A plain-C caller of the ray queries (include/trb.h): it compiles and links against libtrb with nothing but the header, pins
 * the layout of trb_query_ray and trb_intersection, prints every sizeof / offsetof, and prints the status of each entry point
 * called with null arguments (checked before any device is touched, so it runs without a GPU). */
#include <stddef.h>
#include <stdio.h>
#include "trb.h"

_Static_assert(sizeof(trb_query_ray) == 48, "trb_query_ray is 48 bytes");
_Static_assert(offsetof(trb_query_ray, min_t) == 24 && offsetof(trb_query_ray, time) == 32, "trb_query_ray layout");
_Static_assert(sizeof(trb_intersection) == 96, "trb_intersection is 96 bytes");
_Static_assert(offsetof(trb_intersection, p) == 16 && offsetof(trb_intersection, u) == 52 && offsetof(trb_intersection, dp_du) == 64,
               "trb_intersection layout");

#define F(T, f) printf(#T "." #f " %d\n", (int)offsetof(T, f))

int main(void) {
    printf("trb_query_ray sizeof %d\n", (int)sizeof(trb_query_ray));
    F(trb_query_ray, o); F(trb_query_ray, d); F(trb_query_ray, min_t); F(trb_query_ray, max_t); F(trb_query_ray, time); F(trb_query_ray, pad);
    printf("trb_intersection sizeof %d\n", (int)sizeof(trb_intersection));
    F(trb_intersection, t); F(trb_intersection, inst); F(trb_intersection, prim); F(trb_intersection, material); F(trb_intersection, p);
    F(trb_intersection, n); F(trb_intersection, ng); F(trb_intersection, u); F(trb_intersection, v); F(trb_intersection, time);
    F(trb_intersection, dp_du); F(trb_intersection, dp_dv); F(trb_intersection, pad);
    trb_query_ray ray = {{0, 0, 0}, {0, 0, 1}, 0.0f, 1.0f, 0.0f, {0, 0, 0}};
    trb_intersection rec;
    uint8_t occ;
    trb_stats st;
    printf("status trb_intersect_records %d\n", (int)trb_intersect_records(NULL, 1, &ray, &rec, 0, &st));
    printf("status trb_intersect_records_device %d\n", (int)trb_intersect_records_device(NULL, 1, &ray, &rec, 0, NULL, NULL));
    printf("status trb_occluded %d\n", (int)trb_occluded(NULL, 1, &ray, &occ, 0, &st));
    printf("status trb_occluded_device %d\n", (int)trb_occluded_device(NULL, 1, &ray, &occ, 0, NULL, NULL));
    printf("status TRB_INVALID_ARG %d\n", (int)TRB_INVALID_ARG);
    return 0;
}
