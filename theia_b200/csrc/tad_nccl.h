// The ranks' communicator: NCCL for the multi-GPU exchange step, loaded with dlopen so that the library has no link-time
// NCCL dependency (a process that already loaded torch's bundled libnccl.so.2 resolves to that copy; a Go host gets the
// system one), and CUDA IPC for the exported partition buffers.
//
// A loopback group stands in for both when the ranks are contexts of ONE process on one device (tad_debug_loopback_id):
// the collectives copy device to device between the ranks' buffers and a buffer's "IPC handle" is its pointer.  It lets
// the multi-rank paths run on a single GPU.  Its ranks take turns on the device (DESIGN.md section 6).
#pragma once
#include <cstddef>
#include <cstdint>
#include <memory>
#include <cuda_runtime.h>

namespace tad {

struct Loopback;

struct NcclComm {
    void *lib = nullptr;
    void *comm = nullptr;            // the NCCL communicator, or the loopback group
    int world = 1, rank = 0;
    void *fn[8] = {nullptr};
    Loopback *loop = nullptr;        // non-null: a loopback rank (joined through a registered loopback id)
    std::shared_ptr<Loopback> loop_ref;   // the group lives while a rank or the registry holds it
    cudaStream_t streams[3] = {};    // the context's streams: a loopback rank syncs them before it hands the device on
    bool in_job = false;             // loopback: between nccl_job_begin and nccl_job_end
};

int nccl_get_unique_id(void *out, size_t bytes);                 // 128 bytes
int nccl_comm_init(NcclComm *c, int world, int rank, const void *unique_id, size_t bytes);
void nccl_comm_destroy(NcclComm *c);
// byte-granular all-to-all: send_off/send_bytes/recv_off/recv_bytes have `world` entries
int nccl_alltoallv(NcclComm *c, const void *send, const uint64_t *send_off, const uint64_t *send_bytes, void *recv,
                   const uint64_t *recv_off, const uint64_t *recv_bytes, cudaStream_t st);
int nccl_allgather(NcclComm *c, const void *send, void *recv, size_t bytes_per_rank, cudaStream_t st);
// A job's start and end (no-ops for NCCL).  A loopback rank takes the device turn at the start and, after syncing its
// streams, releases it at the end; -1 when the turn did not come within the loopback's wait.
int nccl_job_begin(NcclComm *c);
void nccl_job_end(NcclComm *c);
// CUDA IPC of an exported device buffer through a 64-byte handle (a loopback handle carries the pointer itself)
cudaError_t nccl_ipc_export(NcclComm *c, void *ptr, void *handle);
cudaError_t nccl_ipc_map(NcclComm *c, const void *handle, void **ptr);
cudaError_t nccl_ipc_unmap(NcclComm *c, void *ptr);
const char *nccl_last_error();   // of the calling thread

}  // namespace tad
