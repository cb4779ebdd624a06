// Instantiations of the Hyper-Connections launchers for S = 2 and 3 streams (one file per group so that they compile in
// parallel).
#include "hyper_conn.cuh"

namespace alm {
ALM_HC_INSTANTIATE(template, 2)
ALM_HC_INSTANTIATE(template, 3)
}  // namespace alm
