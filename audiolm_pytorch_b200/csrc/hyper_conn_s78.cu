// Instantiations of the Hyper-Connections launchers for S = 7 and 8 streams (one file per group so that they compile in
// parallel).
#include "hyper_conn.cuh"

namespace alm {
ALM_HC_INSTANTIATE(template, 7)
ALM_HC_INSTANTIATE(template, 8)
}  // namespace alm
