/* A plain-C caller of the moment denoiser (include/trb.h "Moment denoising"): it compiles and links against libtrb with nothing but
 * the header, prints the layout of the two new structs, the two constants, and the status of each entry point called with a null
 * scene or history, null inputs or bad parameters (all checked before any device is touched). */
#include <stddef.h>
#include <stdio.h>
#include "trb.h"

_Static_assert(sizeof(trb_denoise_frame) == 32, "trb_denoise_frame is four pointers");
_Static_assert(sizeof(trb_denoise_moments_output) == 32, "trb_denoise_moments_output is four pointers");

int main(void) {
    printf("trb_denoise_frame sizeof %zu\n", sizeof(trb_denoise_frame));
    printf("trb_denoise_frame.colour %zu\n", offsetof(trb_denoise_frame, colour));
    printf("trb_denoise_frame.albedo_w %zu\n", offsetof(trb_denoise_frame, albedo_w));
    printf("trb_denoise_frame.normal_w %zu\n", offsetof(trb_denoise_frame, normal_w));
    printf("trb_denoise_frame.nearest %zu\n", offsetof(trb_denoise_frame, nearest));
    printf("trb_denoise_moments_output sizeof %zu\n", sizeof(trb_denoise_moments_output));
    printf("trb_denoise_moments_output.rgbw %zu\n", offsetof(trb_denoise_moments_output, rgbw));
    printf("trb_denoise_moments_output.motion %zu\n", offsetof(trb_denoise_moments_output, motion));
    printf("trb_denoise_moments_output.history_length %zu\n", offsetof(trb_denoise_moments_output, history_length));
    printf("trb_denoise_moments_output.variance %zu\n", offsetof(trb_denoise_moments_output, variance));
    printf("const TRB_DENOISE_MOMENTS_MIN_HISTORY %d\n", TRB_DENOISE_MOMENTS_MIN_HISTORY);
    printf("const TRB_DENOISE_MOMENTS_RADIUS %d\n", TRB_DENOISE_MOMENTS_RADIUS);
    float film[16] = {0};
    uint64_t near[4] = {0};
    trb_denoise_frame in = {film, film, film, near};
    trb_denoise_frame no_colour = {NULL, film, film, near};
    trb_denoise_moments_output out = {film, NULL, NULL, NULL};
    trb_denoise_moments_output no_rgbw = {NULL, NULL, NULL, NULL};
    trb_denoise_temporal_params bad = {{5, 128, 4.0f, 1.0f}, 0, 0.05f, 0.9f, 0};
    printf("status trb_denoise_moments:null_scene %d\n", (int)trb_denoise_moments(NULL, NULL, &in, NULL, &out));
    printf("status trb_denoise_moments:null_input %d\n", (int)trb_denoise_moments(NULL, NULL, NULL, NULL, &out));
    printf("status trb_denoise_moments:null_colour %d\n", (int)trb_denoise_moments(NULL, NULL, &no_colour, NULL, &out));
    printf("status trb_denoise_moments:null_rgbw %d\n", (int)trb_denoise_moments(NULL, NULL, &in, NULL, &no_rgbw));
    printf("status trb_denoise_moments:bad_params %d\n", (int)trb_denoise_moments(NULL, NULL, &in, &bad, &out));
    printf("status trb_denoise_moments_device:null_scene %d\n", (int)trb_denoise_moments_device(NULL, NULL, &in, NULL, &out, NULL));
    printf("status trb_denoise_moments_device:bad_params %d\n", (int)trb_denoise_moments_device(NULL, NULL, &in, &bad, &out, NULL));
    printf("status TRB_OK %d\n", (int)TRB_OK);
    printf("status TRB_INVALID_ARG %d\n", (int)TRB_INVALID_ARG);
    return 0;
}
