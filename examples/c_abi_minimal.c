/* Minimal C client of libprisma_b200.so: the drop-in boundary is plain C (no Python, no torch types).
 *
 *   gcc examples/c_abi_minimal.c -Iinclude -Lprisma_b200 -lprisma_b200 -Wl,-rpath,$PWD/prisma_b200 -o /tmp/prisma_c_abi
 *
 * Prints the library version, the transform sizes of every band for a 1080p frame, and shows the error convention:
 * a negative return code plus a thread-local message (here: creating an engine on a machine without an H100).          */
#include <stdio.h>

#include "prisma_b200.h"

int main(void) {
  printf("%s\n", prisma_version());
  const char* bands[4] = {"depth_anything", "depth_anything_metric", "depth_midas", "mask_mmdet"};
  for (int i = 0; i < 4; ++i) {
    int wn = 0, hn = 0;
    if (prisma_net_size(bands[i], 1920, 1080, &wn, &hn) != 0) { printf("error: %s\n", prisma_last_error()); return 1; }
    printf("%-22s 1920x1080 -> %dx%d\n", bands[i], wn, hn);
  }
  int wn, hn;
  if (prisma_net_size("no_such_band", 1920, 1080, &wn, &hn) >= 0) return 2;
  printf("expected error: %s\n", prisma_last_error());
  const int n = prisma_device_count();
  printf("cuda devices: %d\n", n);
  prisma_engine* e = NULL;
  const int rc = prisma_depth_create("vitl", 0, &e);
  if (rc != 0) printf("prisma_depth_create -> %d: %s\n", rc, prisma_last_error());   /* no fallback path: fails loudly */
  else prisma_engine_destroy(e);
  return 0;
}
