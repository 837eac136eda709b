/* A plain-C caller of the denoiser (include/trb.h "Denoising"): it compiles and links against libtrb with nothing but the header,
 * prints the layout of the two denoise structs and the status of each entry point called with a null scene, null inputs or bad
 * parameters (all checked before any device is touched). */
#include <stddef.h>
#include <stdio.h>
#include "trb.h"

_Static_assert(sizeof(trb_denoise_input) == 40, "trb_denoise_input is five pointers");
_Static_assert(sizeof(trb_denoise_params) == 16, "trb_denoise_params is 16 bytes");

int main(void) {
    printf("trb_denoise_input sizeof %zu\n", sizeof(trb_denoise_input));
    printf("trb_denoise_input.colour_a %zu\n", offsetof(trb_denoise_input, colour_a));
    printf("trb_denoise_input.colour_b %zu\n", offsetof(trb_denoise_input, colour_b));
    printf("trb_denoise_input.albedo_w %zu\n", offsetof(trb_denoise_input, albedo_w));
    printf("trb_denoise_input.normal_w %zu\n", offsetof(trb_denoise_input, normal_w));
    printf("trb_denoise_input.nearest %zu\n", offsetof(trb_denoise_input, nearest));
    printf("trb_denoise_params sizeof %zu\n", sizeof(trb_denoise_params));
    printf("trb_denoise_params.iterations %zu\n", offsetof(trb_denoise_params, iterations));
    printf("trb_denoise_params.normal_power %zu\n", offsetof(trb_denoise_params, normal_power));
    printf("trb_denoise_params.sigma_luminance %zu\n", offsetof(trb_denoise_params, sigma_luminance));
    printf("trb_denoise_params.sigma_depth %zu\n", offsetof(trb_denoise_params, sigma_depth));
    float film[16] = {0};
    uint64_t near[4] = {0};
    trb_denoise_input in = {film, film, film, film, near};
    trb_denoise_input no_normal = {film, film, film, NULL, near};
    trb_denoise_params bad = {11, 128, 4.0f, 1.0f};
    printf("status trb_denoise:null_scene %d\n", (int)trb_denoise(NULL, &in, NULL, film));
    printf("status trb_denoise:null_input %d\n", (int)trb_denoise(NULL, NULL, NULL, film));
    printf("status trb_denoise:null_normal %d\n", (int)trb_denoise(NULL, &no_normal, NULL, film));
    printf("status trb_denoise:bad_params %d\n", (int)trb_denoise(NULL, &in, &bad, film));
    printf("status trb_denoise_device:null_scene %d\n", (int)trb_denoise_device(NULL, &in, NULL, film, NULL));
    printf("status trb_denoise_device:bad_params %d\n", (int)trb_denoise_device(NULL, &in, &bad, film, NULL));
    printf("status TRB_INVALID_ARG %d\n", (int)TRB_INVALID_ARG);
    return 0;
}
