/* A plain-C caller of trb_scene_replace_objects (include/trb.h): it compiles and links against libtrb with nothing but the header,
 * prints the layout of trb_scene_objects and the statuses of the null arguments (checked before any device is touched). */
#include <stddef.h>
#include <stdio.h>
#include "trb.h"

#define FIELD(f) printf("offset %s %zu\n", #f, offsetof(trb_scene_objects, f))

int main(void) {
    trb_scene_objects o = {0};
    printf("sizeof trb_scene_objects %zu\n", sizeof(trb_scene_objects));
    FIELD(n_cameras); FIELD(cameras); FIELD(n_instances); FIELD(instances); FIELD(n_splines); FIELD(splines);
    FIELD(n_keyframes); FIELD(keyframes); FIELD(n_knots); FIELD(knots); FIELD(n_color_keys); FIELD(color_keys);
    FIELD(n_fov_floats); FIELD(fov_floats);
    printf("status null_scene %d\n", (int)trb_scene_replace_objects(NULL, &o));
    printf("status null_both %d\n", (int)trb_scene_replace_objects(NULL, NULL));
    printf("status TRB_INVALID_ARG %d\n", (int)TRB_INVALID_ARG);
    return 0;
}
