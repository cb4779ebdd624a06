// Instantiations of the Hyper-Connections launchers for S = 5 and 6 streams (one file per group so that they compile in
// parallel).
#include "hyper_conn.cuh"

namespace alm {
ALM_HC_INSTANTIATE(template, 5)
ALM_HC_INSTANTIATE(template, 6)
}  // namespace alm
