/* A plain-C caller of the scene edit entry points (include/trb.h): it compiles and links against libtrb with nothing but the header,
 * and prints the status of each entry point called with a null scene (checked before any device is touched). */
#include <stdio.h>
#include "trb.h"

int main(void) {
    trb_keyframe kf = {{0, 0, 0}, {0, 0, 0, 1}, {1, 1, 1}};
    trb_color_key ck = {{1, 1, 1, 1}, 0};
    trb_material m = {0};
    printf("status trb_scene_update_keyframes:null_scene %d\n", (int)trb_scene_update_keyframes(NULL, 0, 1, &kf));
    printf("status trb_scene_update_keyframes_device:null_scene %d\n", (int)trb_scene_update_keyframes_device(NULL, 0, 1, &kf, NULL));
    printf("status trb_scene_update_color_keys:null_scene %d\n", (int)trb_scene_update_color_keys(NULL, 0, 1, &ck));
    printf("status trb_scene_update_materials:null_scene %d\n", (int)trb_scene_update_materials(NULL, 0, 1, &m));
    printf("status trb_scene_update_materials:null_scene_empty %d\n", (int)trb_scene_update_materials(NULL, 0, 0, NULL));
    printf("status TRB_INVALID_ARG %d\n", (int)TRB_INVALID_ARG);
    return 0;
}
