/* A plain-C caller of the moment gradients (include/trb.h "Moment gradients"): it compiles and links against libtrb with nothing but
 * the header, prints the layout of the new output struct and the status of each entry point called with a null scene or history,
 * null inputs or outputs, or bad parameters (all checked before any device is touched). */
#include <stddef.h>
#include <stdio.h>
#include "trb.h"

_Static_assert(sizeof(trb_denoise_moments_gradient_output) == 40, "trb_denoise_moments_gradient_output is five pointers");

int main(void) {
    printf("trb_denoise_moments_gradient_output sizeof %zu\n", sizeof(trb_denoise_moments_gradient_output));
    printf("trb_denoise_moments_gradient_output.rgbw %zu\n", offsetof(trb_denoise_moments_gradient_output, rgbw));
    printf("trb_denoise_moments_gradient_output.motion %zu\n", offsetof(trb_denoise_moments_gradient_output, motion));
    printf("trb_denoise_moments_gradient_output.history_length %zu\n", offsetof(trb_denoise_moments_gradient_output, history_length));
    printf("trb_denoise_moments_gradient_output.variance %zu\n", offsetof(trb_denoise_moments_gradient_output, variance));
    printf("trb_denoise_moments_gradient_output.lambda %zu\n", offsetof(trb_denoise_moments_gradient_output, lambda));
    float film[16] = {0}, lam[4] = {0};
    uint64_t near[4] = {0};
    trb_denoise_frame in = {film, film, film, near};
    trb_denoise_frame no_nearest = {film, film, film, NULL};
    trb_denoise_moments_gradient_output out = {film, NULL, NULL, NULL, lam};
    trb_denoise_moments_gradient_output no_rgbw = {NULL, NULL, NULL, NULL, lam};
    trb_denoise_gradient_params bad_iterations = {{{5, 128, 4.0f, 1.0f}, 8, 0.05f, 0.9f, 0}, 7, {0, 0, 0}};
    trb_denoise_gradient_params bad_history = {{{5, 128, 4.0f, 1.0f}, 0, 0.05f, 0.9f, 0}, 3, {0, 0, 0}};
    printf("status trb_denoise_moments_gradient:null_scene %d\n", (int)trb_denoise_moments_gradient(NULL, NULL, &in, NULL, 1, &out));
    printf("status trb_denoise_moments_gradient:null_input %d\n", (int)trb_denoise_moments_gradient(NULL, NULL, NULL, NULL, 1, &out));
    printf("status trb_denoise_moments_gradient:null_nearest %d\n", (int)trb_denoise_moments_gradient(NULL, NULL, &no_nearest, NULL, 1, &out));
    printf("status trb_denoise_moments_gradient:null_output %d\n", (int)trb_denoise_moments_gradient(NULL, NULL, &in, NULL, 1, NULL));
    printf("status trb_denoise_moments_gradient:null_rgbw %d\n", (int)trb_denoise_moments_gradient(NULL, NULL, &in, NULL, 1, &no_rgbw));
    printf("status trb_denoise_moments_gradient:bad_iterations %d\n",
           (int)trb_denoise_moments_gradient(NULL, NULL, &in, &bad_iterations, 1, &out));
    printf("status trb_denoise_moments_gradient:bad_history %d\n", (int)trb_denoise_moments_gradient(NULL, NULL, &in, &bad_history, 1, &out));
    printf("status trb_denoise_moments_gradient_device:null_scene %d\n",
           (int)trb_denoise_moments_gradient_device(NULL, NULL, &in, NULL, 1, &out, NULL));
    printf("status trb_denoise_moments_gradient_device:bad_iterations %d\n",
           (int)trb_denoise_moments_gradient_device(NULL, NULL, &in, &bad_iterations, 1, &out, NULL));
    printf("status trb_denoise_moments_gradient_device:bad_history %d\n",
           (int)trb_denoise_moments_gradient_device(NULL, NULL, &in, &bad_history, 1, &out, NULL));
    printf("status TRB_OK %d\n", (int)TRB_OK);
    printf("status TRB_INVALID_ARG %d\n", (int)TRB_INVALID_ARG);
    return 0;
}
