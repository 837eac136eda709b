/* A plain-C caller of trb_scene_replace_meshes (include/trb.h): it compiles and links against libtrb with nothing but the header,
 * prints the layout of trb_scene_meshes, TRB_MESH_NEW and the statuses of the null arguments (checked before any device is touched). */
#include <stddef.h>
#include <stdio.h>
#include "trb.h"

#define FIELD(f) printf("offset %s %zu\n", #f, offsetof(trb_scene_meshes, f))

int main(void) {
    trb_scene_meshes m = {0};
    printf("sizeof trb_scene_meshes %zu\n", sizeof(trb_scene_meshes));
    FIELD(n_meshes); FIELD(meshes); FIELD(keep);
    printf("const TRB_MESH_NEW %u\n", (unsigned)TRB_MESH_NEW);
    printf("status null_scene %d\n", (int)trb_scene_replace_meshes(NULL, &m, NULL));
    printf("status null_scene_device %d\n", (int)trb_scene_replace_meshes_device(NULL, &m, NULL, NULL));
    printf("status null_both %d\n", (int)trb_scene_replace_meshes(NULL, NULL, NULL));
    printf("status TRB_INVALID_ARG %d\n", (int)TRB_INVALID_ARG);
    return 0;
}
