/* Pins the layout of trb_adaptive (include/trb.h) for plain-C and Rust callers (INTEGRATION.md). */
#include <stddef.h>
#include <stdio.h>
#include "trb.h"

_Static_assert(sizeof(trb_adaptive) == 8, "trb_adaptive is two uint32_t");
_Static_assert(offsetof(trb_adaptive, min_spp) == 0, "min_spp first");
_Static_assert(offsetof(trb_adaptive, max_spp) == 4, "max_spp second");

int main(void) {
    printf("trb_adaptive %zu %zu %zu\n", sizeof(trb_adaptive), offsetof(trb_adaptive, min_spp), offsetof(trb_adaptive, max_spp));
    return 0;
}
