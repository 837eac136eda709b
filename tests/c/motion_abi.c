/* A plain-C caller of the motion-vector calls (include/trb.h "Motion vectors"): it compiles and links against libtrb with nothing but
 * the header, checks trb_motion_sample's size, and prints the status of each entry point called with a null scene (checked before any
 * device is touched). */
#include <stddef.h>
#include <stdio.h>
#include "trb.h"

int main(void) {
    float film[16] = {0};
    trb_render_cfg cfg = {0};
    trb_adaptive ad = {2, 8};
    trb_aov_film aov = {NULL, NULL, NULL};
    trb_sample samples[1];
    trb_aov_sample rec[1];
    trb_motion_sample motion[1];
    printf("size trb_motion_sample %d\n", (int)sizeof(trb_motion_sample));
    printf("status trb_render_aov_motion:null_scene %d\n", (int)trb_render_aov_motion(NULL, &cfg, film, &aov, NULL, film, -0.25f, NULL));
    printf("status trb_render_aov_motion_device:null_scene %d\n",
           (int)trb_render_aov_motion_device(NULL, &cfg, film, &aov, NULL, film, -0.25f, NULL, NULL));
    printf("status trb_render_adaptive_aov_motion:null_scene %d\n",
           (int)trb_render_adaptive_aov_motion(NULL, &cfg, &ad, film, &aov, NULL, film, -0.25f, NULL, NULL));
    printf("status trb_render_adaptive_aov_motion_device:null_scene %d\n",
           (int)trb_render_adaptive_aov_motion_device(NULL, &cfg, &ad, film, &aov, NULL, film, -0.25f, NULL, NULL, NULL));
    printf("status trb_render_samples_aov_motion:null_scene %d\n",
           (int)trb_render_samples_aov_motion(NULL, &cfg, 1, samples, rec, motion, -0.25f, NULL));
    printf("status TRB_OK %d\n", (int)TRB_OK);
    printf("status TRB_INVALID_ARG %d\n", (int)TRB_INVALID_ARG);
    return 0;
}
