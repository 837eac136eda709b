/* A plain-C caller of the variance temporal calls (include/trb.h "Variance temporal denoising"): it compiles and links against libtrb
 * with nothing but the header, and prints the status of each entry point called with a null scene or history, null inputs or outputs,
 * or bad parameters (all checked before any device is touched). */
#include <stddef.h>
#include <stdio.h>
#include "trb.h"

int main(void) {
    float film[16] = {0}, lam[4] = {0};
    uint64_t near[4] = {0};
    trb_denoise_frame in = {film, film, film, near};
    trb_denoise_frame no_colour = {NULL, film, film, near};
    trb_denoise_frame no_albedo = {film, NULL, film, near};
    trb_denoise_frame no_normal = {film, film, NULL, near};
    trb_denoise_frame no_nearest = {film, film, film, NULL};
    trb_denoise_moments_output out = {film, NULL, NULL, NULL};
    trb_denoise_moments_output no_rgbw = {NULL, NULL, NULL, NULL};
    trb_denoise_moments_gradient_output gout = {film, NULL, NULL, NULL, lam};
    trb_denoise_moments_gradient_output gno_rgbw = {NULL, NULL, NULL, NULL, lam};
    trb_denoise_temporal_params bad_history = {{5, 128, 4.0f, 1.0f}, 0, 0.05f, 0.9f, 0};
    trb_denoise_temporal_params bad_spatial = {{11, 128, 4.0f, 1.0f}, 8, 0.05f, 0.9f, 0};
    trb_denoise_gradient_params bad_iterations = {{{5, 128, 4.0f, 1.0f}, 8, 0.05f, 0.9f, 0}, 7, {0, 0, 0}};
    trb_denoise_gradient_params gbad_history = {{{5, 128, 4.0f, 1.0f}, 0, 0.05f, 0.9f, 0}, 3, {0, 0, 0}};
    printf("status trb_denoise_variance_temporal:null_scene %d\n", (int)trb_denoise_variance_temporal(NULL, NULL, &in, film, NULL, &out));
    printf("status trb_denoise_variance_temporal:null_input %d\n", (int)trb_denoise_variance_temporal(NULL, NULL, NULL, film, NULL, &out));
    printf("status trb_denoise_variance_temporal:null_colour %d\n", (int)trb_denoise_variance_temporal(NULL, NULL, &no_colour, film, NULL, &out));
    printf("status trb_denoise_variance_temporal:null_albedo %d\n", (int)trb_denoise_variance_temporal(NULL, NULL, &no_albedo, film, NULL, &out));
    printf("status trb_denoise_variance_temporal:null_normal %d\n", (int)trb_denoise_variance_temporal(NULL, NULL, &no_normal, film, NULL, &out));
    printf("status trb_denoise_variance_temporal:null_nearest %d\n", (int)trb_denoise_variance_temporal(NULL, NULL, &no_nearest, film, NULL, &out));
    printf("status trb_denoise_variance_temporal:null_lum %d\n", (int)trb_denoise_variance_temporal(NULL, NULL, &in, NULL, NULL, &out));
    printf("status trb_denoise_variance_temporal:null_output %d\n", (int)trb_denoise_variance_temporal(NULL, NULL, &in, film, NULL, NULL));
    printf("status trb_denoise_variance_temporal:null_rgbw %d\n", (int)trb_denoise_variance_temporal(NULL, NULL, &in, film, NULL, &no_rgbw));
    printf("status trb_denoise_variance_temporal:bad_history %d\n", (int)trb_denoise_variance_temporal(NULL, NULL, &in, film, &bad_history, &out));
    printf("status trb_denoise_variance_temporal:bad_spatial %d\n", (int)trb_denoise_variance_temporal(NULL, NULL, &in, film, &bad_spatial, &out));
    printf("status trb_denoise_variance_temporal_device:null_scene %d\n",
           (int)trb_denoise_variance_temporal_device(NULL, NULL, &in, film, NULL, &out, NULL));
    printf("status trb_denoise_variance_temporal_device:null_lum %d\n",
           (int)trb_denoise_variance_temporal_device(NULL, NULL, &in, NULL, NULL, &out, NULL));
    printf("status trb_denoise_variance_temporal_device:bad_history %d\n",
           (int)trb_denoise_variance_temporal_device(NULL, NULL, &in, film, &bad_history, &out, NULL));
    printf("status trb_denoise_variance_temporal_gradient:null_scene %d\n",
           (int)trb_denoise_variance_temporal_gradient(NULL, NULL, &in, film, NULL, 1, &gout));
    printf("status trb_denoise_variance_temporal_gradient:null_lum %d\n",
           (int)trb_denoise_variance_temporal_gradient(NULL, NULL, &in, NULL, NULL, 1, &gout));
    printf("status trb_denoise_variance_temporal_gradient:null_output %d\n",
           (int)trb_denoise_variance_temporal_gradient(NULL, NULL, &in, film, NULL, 1, NULL));
    printf("status trb_denoise_variance_temporal_gradient:null_rgbw %d\n",
           (int)trb_denoise_variance_temporal_gradient(NULL, NULL, &in, film, NULL, 1, &gno_rgbw));
    printf("status trb_denoise_variance_temporal_gradient:bad_iterations %d\n",
           (int)trb_denoise_variance_temporal_gradient(NULL, NULL, &in, film, &bad_iterations, 1, &gout));
    printf("status trb_denoise_variance_temporal_gradient:bad_history %d\n",
           (int)trb_denoise_variance_temporal_gradient(NULL, NULL, &in, film, &gbad_history, 1, &gout));
    printf("status trb_denoise_variance_temporal_gradient_device:null_scene %d\n",
           (int)trb_denoise_variance_temporal_gradient_device(NULL, NULL, &in, film, NULL, 1, &gout, NULL));
    printf("status trb_denoise_variance_temporal_gradient_device:null_lum %d\n",
           (int)trb_denoise_variance_temporal_gradient_device(NULL, NULL, &in, NULL, NULL, 1, &gout, NULL));
    printf("status trb_denoise_variance_temporal_gradient_device:bad_iterations %d\n",
           (int)trb_denoise_variance_temporal_gradient_device(NULL, NULL, &in, film, &bad_iterations, 1, &gout, NULL));
    printf("status TRB_OK %d\n", (int)TRB_OK);
    printf("status TRB_INVALID_ARG %d\n", (int)TRB_INVALID_ARG);
    return 0;
}
