/* A plain-C caller of the Adaptive AOV entry points (include/trb.h): it compiles and links against libtrb with nothing but the
 * header and prints the status of each entry point called with a null scene or null buffers (checked before any device is touched). */
#include <stdio.h>
#include "trb.h"

int main(void) {
    trb_render_cfg cfg = {0};
    trb_adaptive ad = {2, 16};
    float film[4] = {0};
    trb_aov_film aov = {0};
    uint32_t spp[1] = {0};
    trb_sample s;
    trb_aov_sample a;
    trb_stats st;
    printf("status trb_render_adaptive_aov:null_scene %d\n", (int)trb_render_adaptive_aov(NULL, &cfg, &ad, film, &aov, spp, &st));
    printf("status trb_render_adaptive_aov:null_adaptive %d\n", (int)trb_render_adaptive_aov(NULL, &cfg, NULL, film, &aov, spp, &st));
    printf("status trb_render_adaptive_aov:null_aov %d\n", (int)trb_render_adaptive_aov(NULL, &cfg, &ad, film, NULL, spp, &st));
    printf("status trb_render_adaptive_aov_device:null_scene %d\n", (int)trb_render_adaptive_aov_device(NULL, &cfg, &ad, film, &aov, NULL, NULL, NULL));
    printf("status trb_render_samples_adaptive_aov:null_scene %d\n", (int)trb_render_samples_adaptive_aov(NULL, &cfg, &ad, 1, &s, &a, spp, &st));
    printf("status trb_render_samples_adaptive_aov:null_buffers %d\n", (int)trb_render_samples_adaptive_aov(NULL, &cfg, &ad, 1, NULL, NULL, spp, &st));
    printf("status TRB_INVALID_ARG %d\n", (int)TRB_INVALID_ARG);
    return 0;
}
