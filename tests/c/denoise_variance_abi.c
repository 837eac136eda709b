/* A plain-C caller of the sample-variance calls (include/trb.h "Sample variance"): it compiles and links against libtrb with nothing
 * but the header, and prints the status of each entry point called with a null scene, null inputs or bad parameters (all checked
 * before any device is touched). */
#include <stddef.h>
#include <stdio.h>
#include "trb.h"

int main(void) {
    float film[16] = {0};
    uint64_t near[4] = {0};
    trb_denoise_frame in = {film, film, film, near};
    trb_denoise_frame no_albedo = {film, NULL, film, near};
    trb_denoise_params bad = {11, 128, 4.0f, 1.0f};
    trb_render_cfg cfg = {0};
    trb_adaptive ad = {2, 8};
    trb_aov_film aov = {NULL, NULL, NULL};
    printf("status trb_denoise_variance:null_scene %d\n", (int)trb_denoise_variance(NULL, &in, film, NULL, film, NULL));
    printf("status trb_denoise_variance:null_input %d\n", (int)trb_denoise_variance(NULL, NULL, film, NULL, film, NULL));
    printf("status trb_denoise_variance:null_albedo %d\n", (int)trb_denoise_variance(NULL, &no_albedo, film, NULL, film, NULL));
    printf("status trb_denoise_variance:null_lum %d\n", (int)trb_denoise_variance(NULL, &in, NULL, NULL, film, NULL));
    printf("status trb_denoise_variance:null_rgbw %d\n", (int)trb_denoise_variance(NULL, &in, film, NULL, NULL, NULL));
    printf("status trb_denoise_variance:bad_params %d\n", (int)trb_denoise_variance(NULL, &in, film, &bad, film, NULL));
    printf("status trb_denoise_variance_device:null_scene %d\n", (int)trb_denoise_variance_device(NULL, &in, film, NULL, film, NULL, NULL));
    printf("status trb_denoise_variance_device:bad_params %d\n", (int)trb_denoise_variance_device(NULL, &in, film, &bad, film, NULL, NULL));
    printf("status trb_render_aov_lum:null_scene %d\n", (int)trb_render_aov_lum(NULL, &cfg, film, &aov, film, NULL));
    printf("status trb_render_aov_lum_device:null_scene %d\n", (int)trb_render_aov_lum_device(NULL, &cfg, film, &aov, film, NULL, NULL));
    printf("status trb_render_adaptive_aov_lum:null_scene %d\n", (int)trb_render_adaptive_aov_lum(NULL, &cfg, &ad, film, &aov, film, NULL, NULL));
    printf("status trb_render_adaptive_aov_lum_device:null_scene %d\n",
           (int)trb_render_adaptive_aov_lum_device(NULL, &cfg, &ad, film, &aov, film, NULL, NULL, NULL));
    printf("status TRB_OK %d\n", (int)TRB_OK);
    printf("status TRB_INVALID_ARG %d\n", (int)TRB_INVALID_ARG);
    return 0;
}
