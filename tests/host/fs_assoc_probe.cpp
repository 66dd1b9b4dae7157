// host probe of fs_assoc_d2 (include/fs2_math.h), the association metric the CUDA kernel evaluates; compiled with g++ by
// tests/test_fs2_assoc_oracle.py and compared with the oracle's restatement (tests/host/fs2_assoc_oracle.c).
#include "../../include/fs2_math.h"

extern "C" int fs_assoc_probe(const double* lm6, const double* pose3, double z0, double z1, double r00, double r11, double* d2) {
    const FsLm L = { lm6[0], lm6[1], lm6[2], lm6[3], lm6[4], lm6[5] };
    return fs_assoc_d2(&L, pose3[0], pose3[1], pose3[2], z0, z1, r00, r11, d2);
}
