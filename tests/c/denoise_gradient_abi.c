/* A plain-C caller of the temporal gradients (include/trb.h "Temporal gradients"): it compiles and links against libtrb with nothing
 * but the header, prints the layout of the two new structs and the status of each entry point called with a null scene or history,
 * null inputs or bad parameters (all checked before any device is touched). */
#include <stddef.h>
#include <stdio.h>
#include "trb.h"

_Static_assert(sizeof(trb_denoise_gradient_params) == 48, "trb_denoise_gradient_params is 48 bytes");
_Static_assert(sizeof(trb_denoise_gradient_output) == 32, "trb_denoise_gradient_output is four pointers");

int main(void) {
    printf("trb_denoise_gradient_params sizeof %zu\n", sizeof(trb_denoise_gradient_params));
    printf("trb_denoise_gradient_params.temporal %zu\n", offsetof(trb_denoise_gradient_params, temporal));
    printf("trb_denoise_gradient_params.iterations %zu\n", offsetof(trb_denoise_gradient_params, iterations));
    printf("trb_denoise_gradient_params.pad %zu\n", offsetof(trb_denoise_gradient_params, pad));
    printf("trb_denoise_gradient_output sizeof %zu\n", sizeof(trb_denoise_gradient_output));
    printf("trb_denoise_gradient_output.rgbw %zu\n", offsetof(trb_denoise_gradient_output, rgbw));
    printf("trb_denoise_gradient_output.motion %zu\n", offsetof(trb_denoise_gradient_output, motion));
    printf("trb_denoise_gradient_output.history_length %zu\n", offsetof(trb_denoise_gradient_output, history_length));
    printf("trb_denoise_gradient_output.lambda %zu\n", offsetof(trb_denoise_gradient_output, lambda));
    float film[16] = {0};
    uint64_t near[4] = {0};
    trb_denoise_input in = {film, film, film, film, near};
    trb_denoise_gradient_output out = {film, NULL, NULL, NULL};
    trb_denoise_gradient_output no_rgbw = {NULL, NULL, NULL, NULL};
    trb_denoise_gradient_params bad = {{{5, 128, 4.0f, 1.0f}, 8, 0.05f, 0.9f, 0}, 7, {0, 0, 0}};
    trb_denoise_gradient_params bad_temporal = {{{5, 128, 4.0f, 1.0f}, 0, 0.05f, 0.9f, 0}, 3, {0, 0, 0}};
    printf("status trb_denoise_temporal_gradient:null_scene %d\n", (int)trb_denoise_temporal_gradient(NULL, NULL, &in, NULL, 1, &out));
    printf("status trb_denoise_temporal_gradient:null_input %d\n", (int)trb_denoise_temporal_gradient(NULL, NULL, NULL, NULL, 1, &out));
    printf("status trb_denoise_temporal_gradient:null_output %d\n", (int)trb_denoise_temporal_gradient(NULL, NULL, &in, NULL, 1, NULL));
    printf("status trb_denoise_temporal_gradient:null_rgbw %d\n", (int)trb_denoise_temporal_gradient(NULL, NULL, &in, NULL, 1, &no_rgbw));
    printf("status trb_denoise_temporal_gradient:bad_iterations %d\n", (int)trb_denoise_temporal_gradient(NULL, NULL, &in, &bad, 1, &out));
    printf("status trb_denoise_temporal_gradient:bad_temporal %d\n", (int)trb_denoise_temporal_gradient(NULL, NULL, &in, &bad_temporal, 1, &out));
    printf("status trb_denoise_temporal_gradient_device:null_scene %d\n",
           (int)trb_denoise_temporal_gradient_device(NULL, NULL, &in, NULL, 1, &out, NULL));
    printf("status trb_denoise_temporal_gradient_device:bad_iterations %d\n",
           (int)trb_denoise_temporal_gradient_device(NULL, NULL, &in, &bad, 1, &out, NULL));
    printf("status TRB_OK %d\n", (int)TRB_OK);
    printf("status TRB_INVALID_ARG %d\n", (int)TRB_INVALID_ARG);
    return 0;
}
