/* A plain-C caller of the AOV entry points (include/trb.h): it compiles and links against libtrb with nothing but the header, prints
 * the layout of the two AOV structs, and the status of each entry point called with a null scene or null buffers (checked before any
 * device is touched). */
#include <stddef.h>
#include <stdio.h>
#include "trb.h"

_Static_assert(sizeof(trb_aov_sample) == 32, "trb_aov_sample is 32 bytes");
_Static_assert(sizeof(trb_aov_film) == 24, "trb_aov_film is three pointers");

int main(void) {
    printf("trb_aov_sample sizeof %zu\n", sizeof(trb_aov_sample));
    printf("trb_aov_sample.albedo %zu\n", offsetof(trb_aov_sample, albedo));
    printf("trb_aov_sample.depth %zu\n", offsetof(trb_aov_sample, depth));
    printf("trb_aov_sample.n %zu\n", offsetof(trb_aov_sample, n));
    printf("trb_aov_sample.inst %zu\n", offsetof(trb_aov_sample, inst));
    printf("trb_aov_film sizeof %zu\n", sizeof(trb_aov_film));
    printf("trb_aov_film.albedo_w %zu\n", offsetof(trb_aov_film, albedo_w));
    printf("trb_aov_film.normal_w %zu\n", offsetof(trb_aov_film, normal_w));
    printf("trb_aov_film.nearest %zu\n", offsetof(trb_aov_film, nearest));
    trb_render_cfg cfg = {0};
    float film[4] = {0};
    trb_aov_film aov = {0};
    trb_sample s;
    trb_aov_sample a;
    trb_stats st;
    printf("status trb_render_aov:null_scene %d\n", (int)trb_render_aov(NULL, &cfg, film, &aov, &st));
    printf("status trb_render_aov:null_cfg %d\n", (int)trb_render_aov(NULL, NULL, film, &aov, &st));
    printf("status trb_render_aov_device:null_scene %d\n", (int)trb_render_aov_device(NULL, &cfg, film, &aov, NULL, NULL));
    printf("status trb_render_samples_aov:null_scene %d\n", (int)trb_render_samples_aov(NULL, &cfg, 1, &s, &a, &st));
    printf("status trb_render_samples_aov:null_buffers %d\n", (int)trb_render_samples_aov(NULL, &cfg, 1, NULL, NULL, &st));
    printf("status TRB_INVALID_ARG %d\n", (int)TRB_INVALID_ARG);
    return 0;
}
