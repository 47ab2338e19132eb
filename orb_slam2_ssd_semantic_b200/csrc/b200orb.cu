// b200orb.cu -- single translation unit of libb200orb.so (kernels live in headers shared by the parts below).
#include "orbx.cu"
#include "orbm.cu"
#include "orbs.cu"
#include "ocm.cu"
#include "gcm.cu"
#include "orbv.cu"
#include "dynm.cu"
#include "orbv_db.cu"
