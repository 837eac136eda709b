/* A plain-C caller of trb_scene_replace_settings and trb_scene_replace_materials (include/trb.h): it compiles and links against libtrb
 * with nothing but the header, prints the layouts of trb_scene_materials, trb_film and trb_integrator and the statuses of the null
 * arguments (checked before any device is touched). */
#include <stddef.h>
#include <stdio.h>
#include "trb.h"

#define FIELD(f) printf("offset %s %zu\n", #f, offsetof(trb_scene_materials, f))

int main(void) {
    trb_scene_materials m = {0};
    trb_film film = {0};
    trb_integrator integrator = {0};
    printf("sizeof trb_scene_materials %zu\n", sizeof(trb_scene_materials));
    printf("sizeof trb_film %zu\n", sizeof(trb_film));
    printf("sizeof trb_integrator %zu\n", sizeof(trb_integrator));
    FIELD(n_materials); FIELD(materials); FIELD(n_merl); FIELD(merl_tables); FIELD(n_textures); FIELD(textures); FIELD(n_images); FIELD(images);
    printf("status settings_null_scene %d\n", (int)trb_scene_replace_settings(NULL, &film, &integrator));
    printf("status settings_all_null %d\n", (int)trb_scene_replace_settings(NULL, NULL, NULL));
    printf("status materials_null_scene %d\n", (int)trb_scene_replace_materials(NULL, &m, NULL));
    printf("status materials_null_scene_device %d\n", (int)trb_scene_replace_materials_device(NULL, &m, NULL, NULL));
    printf("status materials_null_both %d\n", (int)trb_scene_replace_materials(NULL, NULL, NULL));
    printf("status TRB_INVALID_ARG %d\n", (int)TRB_INVALID_ARG);
    return 0;
}
