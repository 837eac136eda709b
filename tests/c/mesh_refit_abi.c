/* A plain-C caller of the mesh refit entry points (include/trb.h): it compiles and links against libtrb with nothing but the header,
 * and prints the status of each entry point called with a null scene (checked before any device is touched). */
#include <stdio.h>
#include "trb.h"

int main(void) {
    float v[9] = {0, 0, 0, 1, 0, 0, 0, 1, 0};
    printf("status trb_scene_refit_mesh:null_scene %d\n", (int)trb_scene_refit_mesh(NULL, 0, v, v, v));
    printf("status trb_scene_refit_mesh:null_positions %d\n", (int)trb_scene_refit_mesh(NULL, 0, NULL, v, NULL));
    printf("status trb_scene_refit_mesh:null_all %d\n", (int)trb_scene_refit_mesh(NULL, 0, NULL, NULL, NULL));
    printf("status trb_scene_refit_mesh_device:null_scene %d\n", (int)trb_scene_refit_mesh_device(NULL, 0, v, NULL, NULL, NULL));
    printf("status trb_scene_refit_mesh_device:null_all %d\n", (int)trb_scene_refit_mesh_device(NULL, 3, NULL, NULL, NULL, NULL));
    printf("status TRB_INVALID_ARG %d\n", (int)TRB_INVALID_ARG);
    return 0;
}
