/* A plain-C caller of the multi-GPU AOV entry points (include/trb.h): it compiles and links against libtrb with nothing but the
 * header, and prints the status of each entry point called with null arguments (checked before any device is touched, so it runs
 * without a GPU). */
#include <stdio.h>
#include "trb.h"

int main(void) {
    trb_render_cfg cfg = {0};
    trb_adaptive ad = {2, 32};
    float film[4] = {0}, albedo[4] = {0}, normal[4] = {0};
    uint64_t nearest[1] = {~0ull};
    trb_aov_film aov = {albedo, normal, nearest};
    uint32_t spp[1] = {0};
    trb_stats st;
    printf("trb_render_sharded_aov %d\n", (int)trb_render_sharded_aov(NULL, NULL, &cfg, 0, film, &aov, &st));
    printf("trb_render_sharded_adaptive_aov %d\n", (int)trb_render_sharded_adaptive_aov(NULL, NULL, &cfg, &ad, 0, film, &aov, spp, &st));
    printf("trb_group_render_aov %d\n", (int)trb_group_render_aov(NULL, &cfg, film, &aov, &st));
    printf("trb_group_render_adaptive_aov %d\n", (int)trb_group_render_adaptive_aov(NULL, &cfg, &ad, film, &aov, spp, &st));
    printf("TRB_INVALID_ARG %d\n", (int)TRB_INVALID_ARG);
    return 0;
}
