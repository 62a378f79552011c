// CUB device scans of the engine that have a translation unit of their own: a new CUB instance in tad_kernels.cu or
// tad_spill.cu would move the constant-bank addresses that every existing kernel of that unit is compiled against.
#include <cub/device/device_scan.cuh>

#include "tad_kernels.h"

namespace tad {

cudaError_t exclusive_scan_u32(void *temp, size_t &temp_bytes, const uint32_t *in, uint32_t *out, int n, cudaStream_t st)
{
    return cub::DeviceScan::ExclusiveSum(temp, temp_bytes, in, out, n, st);
}

}  // namespace tad
