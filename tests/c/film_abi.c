/* A plain-C caller of the film-write and device camera-ray entry points (include/trb.h): it compiles and links against libtrb with
 * nothing but the header, pins trb_sample's layout, and prints the status of each entry point called with null arguments (checked
 * before any device is touched, so it runs without a GPU). */
#include <stddef.h>
#include <stdio.h>
#include "trb.h"

_Static_assert(sizeof(trb_sample) == 20 && offsetof(trb_sample, y) == 4 && offsetof(trb_sample, r) == 8 && offsetof(trb_sample, b) == 16,
               "trb_sample layout");

int main(void) {
    trb_sample s = {0.5f, 0.5f, 1.0f, 1.0f, 1.0f};
    uint32_t region = 0;
    float film[4] = {0};
    trb_render_cfg cfg = {0};
    trb_ray ray;
    float xy[2];
    printf("status trb_film_write %d\n", (int)trb_film_write(NULL, 1, &s, &region, film));
    printf("status trb_film_write_device %d\n", (int)trb_film_write_device(NULL, 1, &s, &region, film, NULL));
    printf("status trb_camera_rays_device %d\n", (int)trb_camera_rays_device(NULL, &cfg, 1, &ray, xy, NULL));
    printf("status TRB_INVALID_ARG %d\n", (int)TRB_INVALID_ARG);
    return 0;
}
