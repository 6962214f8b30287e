/* A plain-C client of the drop-in boundary (include/onepose_b200.h): what a cgo / JNI / FFI stub sees.  Built by
 * tests/test_host_cpu.py with gcc -std=c99 and linked against the in-tree shared library; no C++, no torch, no CUDA headers.
 * Without a GPU every constructor must fail with OPB_E_CUDA and a message (there is no CPU path); with one, a matcher and an
 * extractor are created and destroyed.  Exit code 0 = the behaviour expected for the machine it runs on. */
#include <stdio.h>
#include <string.h>

#include "onepose_b200.h"

int main(void) {
  opb_config cfg;
  opb_sp_config scfg;
  opb_matcher* m = NULL;
  opb_superpoint* s = NULL;
  int rc, rc2;
  memset(&cfg, 0, sizeof cfg);
  cfg.descriptor_dim = 256; cfg.num_heads = 4; cfg.scale_factor = 0.07f; cfg.match_threshold = 0.2f; cfg.include_self = 1;
  memset(&scfg, 0, sizeof scfg);
  scfg.descriptor_dim = 256; scfg.nms_radius = 3; scfg.keypoint_threshold = 0.005f; scfg.max_keypoints = 4096; scfg.remove_borders = 4;
  scfg.align_corners = 1;
  rc = opb_create(&cfg, &m);
  printf("opb_create -> %d (%s)\n", rc, rc ? opb_last_error(NULL) : "ok");
  rc2 = opb_sp_create(&scfg, &s);
  printf("opb_sp_create -> %d (%s)\n", rc2, rc2 ? opb_sp_last_error(NULL) : "ok");
  /* the range guards report nothing for a null handle or one that has not run yet */
  if (opb_sp_poll_range(s) != OPB_OK || opb_sp_check_range(s, NULL) != OPB_OK) return 3;
  if (opb_poll_range(m) != OPB_OK || opb_check_range(m, NULL) != OPB_OK) return 3;
  if (rc == OPB_OK && rc2 == OPB_OK) {            /* GPU box */
    opb_destroy(m);
    opb_sp_destroy(s);
    return 0;
  }
  if (rc == OPB_E_CUDA && rc2 == OPB_E_CUDA && strlen(opb_last_error(NULL)) > 0 && strlen(opb_sp_last_error(NULL)) > 0) return 0;
  return 2;
}
