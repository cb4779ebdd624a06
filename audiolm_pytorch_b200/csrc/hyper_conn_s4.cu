// Instantiations of the Hyper-Connections launchers for S = 4 streams (one file per group so that they compile in
// parallel).
#include "hyper_conn.cuh"

namespace alm {
ALM_HC_INSTANTIATE(template, 4)
}  // namespace alm
