/* A plain-C caller of the BVH build entry points (include/trb.h): it compiles and links against libtrb with nothing but the header,
 * pins trb_bvh_node's layout, and prints the status of each entry point called with null or empty arguments (checked before any
 * device is touched) and with one valid box (TRB_NO_DEVICE without a GPU). */
#include <stddef.h>
#include <stdio.h>
#include "trb.h"

_Static_assert(sizeof(trb_bvh_node) == 32 && offsetof(trb_bvh_node, bmax) == 12 && offsetof(trb_bvh_node, a) == 24 && offsetof(trb_bvh_node, b) == 28,
               "trb_bvh_node layout");

int main(void) {
    float box[6] = {0, 0, 0, 1, 1, 1};
    uint32_t n_nodes = 0, order[1];
    trb_bvh_node nodes[1];
    printf("status trb_build_bvh:null %d\n", (int)trb_build_bvh(0, NULL, 1, 16, &n_nodes, NULL, NULL));
    printf("status trb_build_bvh:empty %d\n", (int)trb_build_bvh(0, box, 0, 16, &n_nodes, NULL, NULL));
    printf("status trb_build_bvh_device:null %d\n", (int)trb_build_bvh_device(0, box, 1, 16, NULL, nodes, order, NULL));
    printf("status trb_build_bvh_device:empty %d\n", (int)trb_build_bvh_device(0, box, 0, 16, &n_nodes, nodes, order, NULL));
    printf("status trb_build_bvh:one %d\n", (int)trb_build_bvh(0, box, 1, 16, &n_nodes, nodes, order));
    printf("status TRB_INVALID_ARG %d\n", (int)TRB_INVALID_ARG);
    printf("status TRB_NO_DEVICE %d\n", (int)TRB_NO_DEVICE);
    return 0;
}
