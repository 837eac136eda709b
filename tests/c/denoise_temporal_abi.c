/* A plain-C caller of the temporal denoiser (include/trb.h "Temporal denoising"): it compiles and links against libtrb with nothing
 * but the header, prints the layout of the two new structs and the status of each entry point called with a null scene or history,
 * null inputs or bad parameters (all checked before any device is touched). */
#include <stddef.h>
#include <stdio.h>
#include "trb.h"

_Static_assert(sizeof(trb_denoise_temporal_params) == 32, "trb_denoise_temporal_params is 32 bytes");
_Static_assert(sizeof(trb_denoise_temporal_output) == 24, "trb_denoise_temporal_output is three pointers");

int main(void) {
    printf("trb_denoise_temporal_params sizeof %zu\n", sizeof(trb_denoise_temporal_params));
    printf("trb_denoise_temporal_params.spatial %zu\n", offsetof(trb_denoise_temporal_params, spatial));
    printf("trb_denoise_temporal_params.max_history %zu\n", offsetof(trb_denoise_temporal_params, max_history));
    printf("trb_denoise_temporal_params.depth_tolerance %zu\n", offsetof(trb_denoise_temporal_params, depth_tolerance));
    printf("trb_denoise_temporal_params.normal_threshold %zu\n", offsetof(trb_denoise_temporal_params, normal_threshold));
    printf("trb_denoise_temporal_params.pad %zu\n", offsetof(trb_denoise_temporal_params, pad));
    printf("trb_denoise_temporal_output sizeof %zu\n", sizeof(trb_denoise_temporal_output));
    printf("trb_denoise_temporal_output.rgbw %zu\n", offsetof(trb_denoise_temporal_output, rgbw));
    printf("trb_denoise_temporal_output.motion %zu\n", offsetof(trb_denoise_temporal_output, motion));
    printf("trb_denoise_temporal_output.history_length %zu\n", offsetof(trb_denoise_temporal_output, history_length));
    float film[16] = {0};
    uint64_t near[4] = {0};
    trb_denoise_input in = {film, film, film, film, near};
    trb_denoise_temporal_output out = {film, NULL, NULL};
    trb_denoise_temporal_output no_rgbw = {NULL, NULL, NULL};
    trb_denoise_temporal_params bad = {{5, 128, 4.0f, 1.0f}, 0, 0.05f, 0.9f, 0};
    trb_denoise_history* h = NULL;
    printf("status trb_denoise_history_create:null_scene %d\n", (int)trb_denoise_history_create(NULL, &h));
    printf("status trb_denoise_history_reset:null %d\n", (int)trb_denoise_history_reset(NULL));
    printf("status trb_denoise_history_destroy:null %d\n", (int)trb_denoise_history_destroy(NULL));
    printf("status trb_denoise_temporal:null_scene %d\n", (int)trb_denoise_temporal(NULL, NULL, &in, NULL, &out));
    printf("status trb_denoise_temporal:null_input %d\n", (int)trb_denoise_temporal(NULL, NULL, NULL, NULL, &out));
    printf("status trb_denoise_temporal:null_rgbw %d\n", (int)trb_denoise_temporal(NULL, NULL, &in, NULL, &no_rgbw));
    printf("status trb_denoise_temporal:bad_params %d\n", (int)trb_denoise_temporal(NULL, NULL, &in, &bad, &out));
    printf("status trb_denoise_temporal_device:null_scene %d\n", (int)trb_denoise_temporal_device(NULL, NULL, &in, NULL, &out, NULL));
    printf("status trb_denoise_temporal_device:bad_params %d\n", (int)trb_denoise_temporal_device(NULL, NULL, &in, &bad, &out, NULL));
    printf("status TRB_OK %d\n", (int)TRB_OK);
    printf("status TRB_INVALID_ARG %d\n", (int)TRB_INVALID_ARG);
    return 0;
}
