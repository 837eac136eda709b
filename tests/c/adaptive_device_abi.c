/* A plain-C caller of the Adaptive sampler's stream-ordered and multi-GPU entry points (include/trb.h): it compiles and
 * links against libtrb with nothing but the header, and prints the status of each entry point called with null arguments
 * (checked before any device is touched, so it runs without a GPU). */
#include <stdio.h>
#include "trb.h"

int main(void) {
    trb_render_cfg cfg = {0};
    trb_adaptive ad = {2, 32};
    float film[4] = {0};
    uint32_t spp[1] = {0};
    trb_stats st;
    printf("trb_render_adaptive_device %d\n", (int)trb_render_adaptive_device(NULL, &cfg, &ad, film, NULL, NULL, NULL));
    printf("trb_render_sharded_adaptive %d\n", (int)trb_render_sharded_adaptive(NULL, NULL, &cfg, &ad, 0, film, spp, &st));
    printf("trb_group_render_adaptive %d\n", (int)trb_group_render_adaptive(NULL, &cfg, &ad, film, spp, &st));
    printf("TRB_INVALID_ARG %d\n", (int)TRB_INVALID_ARG);
    return 0;
}
