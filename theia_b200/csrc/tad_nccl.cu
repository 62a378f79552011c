#include "tad_nccl.h"

#include <dlfcn.h>

#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <random>

namespace tad {
namespace {

struct UniqueId { char internal[128]; };
typedef int (*fn_get_uid)(UniqueId *);
typedef int (*fn_init_rank)(void **, int, UniqueId, int);
typedef int (*fn_destroy)(void *);
typedef int (*fn_send)(const void *, size_t, int, int, void *, cudaStream_t);
typedef int (*fn_recv)(void *, size_t, int, int, void *, cudaStream_t);
typedef int (*fn_group)(void);
typedef int (*fn_allgather)(const void *, void *, size_t, int, void *, cudaStream_t);
typedef const char *(*fn_errstr)(int);

thread_local char g_err[256] = "";   // every rank of a loopback group is a thread of this process
void *g_lib = nullptr;

void *open_lib()
{
    if (g_lib) return g_lib;
    const char *names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char *n : names) {
        g_lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
        if (g_lib) return g_lib;
    }
    snprintf(g_err, sizeof(g_err), "cannot load libnccl.so.2: %s", dlerror());
    return nullptr;
}

void *sym(void *lib, const char *name)
{
    void *p = dlsym(lib, name);
    if (!p) snprintf(g_err, sizeof(g_err), "missing NCCL symbol %s", name);
    return p;
}

enum { F_INIT = 0, F_DESTROY, F_SEND, F_RECV, F_GSTART, F_GEND, F_ALLGATHER, F_ERRSTR };
constexpr int kNcclInt8 = 0;   // ncclInt8 / ncclChar

int check(NcclComm *c, int rc, const char *what)
{
    if (rc == 0) return 0;
    const char *s = c->fn[F_ERRSTR] ? ((fn_errstr)c->fn[F_ERRSTR])(rc) : "?";
    snprintf(g_err, sizeof(g_err), "%s failed: %s", what, s);
    return -1;
}


// ---- loopback group: W ranks as contexts of one process on one device ------------------------------------------------
constexpr int kLoopRanks = 8;
constexpr auto kLoopWait = std::chrono::seconds(300);     // bounds every rendezvous and every wait for the device turn
constexpr char kLoopMagic[16] = "tad-loopback-id";         // 15 characters + NUL

// What a rank brings to the collective in progress; its peers read it between the two rendezvous.
struct Post {
    const void *send = nullptr;
    size_t bytes = 0;                                       // allgather: bytes per rank
    const uint64_t *send_off = nullptr, *send_bytes = nullptr;     // alltoallv
};

}  // namespace

struct Loopback {
    int world = 0;
    uint64_t token = 0;
    std::mutex mu;
    std::condition_variable cv;
    bool member[kLoopRanks] = {};
    int joined = 0;
    uint64_t gen = 0;              // rendezvous generation
    int arrived = 0;
    bool here[kLoopRanks] = {};
    Post post[kLoopRanks];
    int turn = -1;                 // the rank that may run device work, -1: none
};

namespace {

std::mutex g_reg_mu;
// groups registered by tad_debug_loopback_id and still open to joins: a group leaves the registry when its last rank
// joins or when tad_debug_loopback_release drops its id; the ranks that joined keep it alive
std::map<uint64_t, std::shared_ptr<Loopback>> g_reg;

// The registered group an id names, or null (any id that tad_debug_loopback_id did not write in this process).
std::shared_ptr<Loopback> loop_lookup(const void *id)
{
    if (memcmp(id, kLoopMagic, sizeof(kLoopMagic)) != 0) return nullptr;
    uint64_t token;
    memcpy(&token, static_cast<const char *>(id) + 16, 8);
    std::lock_guard<std::mutex> lk(g_reg_mu);
    auto it = g_reg.find(token);
    return it == g_reg.end() ? nullptr : it->second;
}

// Waits until every rank of the group has arrived (lock held).  On timeout names the ranks that did not.
int rendezvous(Loopback *g, int me, std::unique_lock<std::mutex> &lk)
{
    const uint64_t gen = g->gen;
    g->here[me] = true;
    if (++g->arrived == g->world) {
        g->arrived = 0;
        for (bool &h : g->here) h = false;
        g->gen++;
        g->cv.notify_all();
        return 0;
    }
    if (g->cv.wait_for(lk, kLoopWait, [&] { return g->gen != gen; })) return 0;
    g->arrived--;
    g->here[me] = false;
    int n = snprintf(g_err, sizeof(g_err), "loopback rank %d: ranks", me);
    for (int r = 0; r < g->world; r++)
        if (r != me && !g->here[r] && n < (int)sizeof(g_err)) n += snprintf(g_err + n, sizeof(g_err) - n, " %d", r);
    if (n < (int)sizeof(g_err))
        snprintf(g_err + n, sizeof(g_err) - n, " did not reach the collective within %d s", (int)kLoopWait.count());
    return -1;
}

int take_turn(Loopback *g, int me)
{
    std::unique_lock<std::mutex> lk(g->mu);
    if (!g->cv.wait_for(lk, kLoopWait, [&] { return g->turn < 0 || g->turn == me; })) {
        snprintf(g_err, sizeof(g_err), "loopback rank %d: rank %d held the device turn for more than %d s", me, g->turn,
                 (int)kLoopWait.count());
        return -1;
    }
    g->turn = me;
    return 0;
}

void release_turn(Loopback *g, int me)
{
    std::lock_guard<std::mutex> lk(g->mu);
    if (g->turn == me) {
        g->turn = -1;
        g->cv.notify_all();
    }
}

int sync_streams(NcclComm *c, cudaStream_t st)
{
    for (cudaStream_t s : {c->streams[0], c->streams[1], c->streams[2], st}) {
        const cudaError_t e = s ? cudaStreamSynchronize(s) : cudaSuccess;
        if (e != cudaSuccess) {
            snprintf(g_err, sizeof(g_err), "loopback rank %d: %s", c->rank, cudaGetErrorString(e));
            return -1;
        }
    }
    return 0;
}

// One loopback collective.  Entering it, the rank finishes its device work and hands the device turn on; the ranks meet;
// `copy` pulls the peers' data (their posts are stable until the second meeting) on `st`, which is synced; the ranks
// meet again, so no rank reuses a buffer a peer still reads; leaving, a rank inside a job takes the turn again.
template <class F>
int loop_collective(NcclComm *c, const Post &mine, cudaStream_t st, F &&copy)
{
    Loopback *g = c->loop;
    const int me = c->rank;
    if (sync_streams(c, st)) return -1;
    if (c->in_job) release_turn(g, me);
    {
        std::unique_lock<std::mutex> lk(g->mu);
        g->post[me] = mine;
        if (rendezvous(g, me, lk)) return -1;
    }
    int rc = copy(g);
    if (rc == 0) {
        const cudaError_t e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) {
            snprintf(g_err, sizeof(g_err), "loopback rank %d: %s", me, cudaGetErrorString(e));
            rc = -1;
        }
    }
    {
        std::unique_lock<std::mutex> lk(g->mu);      // the peers wait here whatever this rank's copy did
        if (rendezvous(g, me, lk)) return -1;
    }
    if (rc == 0 && c->in_job) rc = take_turn(g, me);
    return rc;
}

int copy_err(int me, cudaError_t e)
{
    snprintf(g_err, sizeof(g_err), "loopback rank %d: %s", me, cudaGetErrorString(e));
    return -1;
}

int loop_allgather(NcclComm *c, const void *send, void *recv, size_t bytes, cudaStream_t st)
{
    Post mine;
    mine.send = send;
    mine.bytes = bytes;
    return loop_collective(c, mine, st, [&](Loopback *g) {
        for (int p = 0; p < c->world; p++) {
            if (g->post[p].bytes != bytes) {
                snprintf(g_err, sizeof(g_err), "loopback all-gather: rank %d sends %zu bytes, rank %d %zu", p,
                         g->post[p].bytes, c->rank, bytes);
                return -1;
            }
            const cudaError_t e = cudaMemcpyAsync(static_cast<char *>(recv) + p * bytes, g->post[p].send, bytes,
                                                  cudaMemcpyDeviceToDevice, st);
            if (e != cudaSuccess) return copy_err(c->rank, e);
        }
        return 0;
    });
}

int loop_alltoallv(NcclComm *c, const void *send, const uint64_t *send_off, const uint64_t *send_bytes, void *recv,
                   const uint64_t *recv_off, const uint64_t *recv_bytes, cudaStream_t st)
{
    Post mine;
    mine.send = send;
    mine.send_off = send_off;
    mine.send_bytes = send_bytes;
    const int me = c->rank;
    return loop_collective(c, mine, st, [&](Loopback *g) {
        for (int p = 0; p < c->world; p++) {
            if (p == me) continue;                 // as with NCCL: a rank's own rows stay where they are
            const uint64_t n = g->post[p].send_bytes[me];
            if (n != recv_bytes[p]) {
                snprintf(g_err, sizeof(g_err), "loopback all-to-all: rank %d sends %llu bytes to rank %d, which expects %llu",
                         p, (unsigned long long)n, me, (unsigned long long)recv_bytes[p]);
                return -1;
            }
            if (!n) continue;
            const cudaError_t e = cudaMemcpyAsync(static_cast<char *>(recv) + recv_off[p],
                                                  static_cast<const char *>(g->post[p].send) + g->post[p].send_off[me], n,
                                                  cudaMemcpyDeviceToDevice, st);
            if (e != cudaSuccess) return copy_err(me, e);
        }
        return 0;
    });
}

int loop_join(NcclComm *c, std::shared_ptr<Loopback> g, int world, int rank)
{
    std::unique_lock<std::mutex> lk(g->mu);
    if (g->world != world || rank < 0 || rank >= world || g->member[rank]) {
        snprintf(g_err, sizeof(g_err), "loopback id of %d ranks: cannot join as rank %d of %d%s", g->world, rank, world,
                 rank >= 0 && rank < g->world && g->member[rank] ? " (taken)" : "");
        return -1;
    }
    g->member[rank] = true;
    const bool all = ++g->joined == g->world;
    c->loop = g.get();
    c->loop_ref = g;
    c->comm = g.get();
    c->world = world;
    c->rank = rank;
    lk.unlock();
    if (all) {
        std::lock_guard<std::mutex> rl(g_reg_mu);
        g_reg.erase(g->token);            // every rank is in: nobody else may join
    }
    return 0;
}

}  // namespace

const char *nccl_last_error() { return g_err; }

int nccl_get_unique_id(void *out, size_t bytes)
{
    if (bytes < sizeof(UniqueId)) return -1;
    void *lib = open_lib();
    if (!lib) return -1;
    fn_get_uid f = (fn_get_uid)sym(lib, "ncclGetUniqueId");
    if (!f) return -1;
    UniqueId id;
    if (f(&id) != 0) { snprintf(g_err, sizeof(g_err), "ncclGetUniqueId failed"); return -1; }
    memcpy(out, &id, sizeof(id));
    return 0;
}

int nccl_comm_init(NcclComm *c, int world, int rank, const void *unique_id, size_t bytes)
{
    if (!unique_id || bytes < sizeof(UniqueId)) { snprintf(g_err, sizeof(g_err), "missing ncclUniqueId"); return -1; }
    // a loopback id selects the loopback only while its group is registered in this process
    if (std::shared_ptr<Loopback> g = loop_lookup(unique_id)) return loop_join(c, g, world, rank);
    c->lib = open_lib();
    if (!c->lib) return -1;
    const char *names[8] = {"ncclCommInitRank", "ncclCommDestroy", "ncclSend", "ncclRecv", "ncclGroupStart",
                            "ncclGroupEnd", "ncclAllGather", "ncclGetErrorString"};
    for (int i = 0; i < 8; i++) {
        c->fn[i] = sym(c->lib, names[i]);
        if (!c->fn[i]) return -1;
    }
    UniqueId id;
    memcpy(&id, unique_id, sizeof(id));
    c->world = world;
    c->rank = rank;
    return check(c, ((fn_init_rank)c->fn[F_INIT])(&c->comm, world, id, rank), "ncclCommInitRank");
}

void nccl_comm_destroy(NcclComm *c)
{
    if (c->loop) {
        nccl_job_end(c);
        c->loop = nullptr;
        c->loop_ref.reset();              // the last rank out frees the group
        c->comm = nullptr;
        return;
    }
    if (c->comm && c->fn[F_DESTROY]) ((fn_destroy)c->fn[F_DESTROY])(c->comm);
    c->comm = nullptr;
}

int nccl_alltoallv(NcclComm *c, const void *send, const uint64_t *send_off, const uint64_t *send_bytes, void *recv,
                   const uint64_t *recv_off, const uint64_t *recv_bytes, cudaStream_t st)
{
    if (c->loop) return loop_alltoallv(c, send, send_off, send_bytes, recv, recv_off, recv_bytes, st);
    if (check(c, ((fn_group)c->fn[F_GSTART])(), "ncclGroupStart")) return -1;
    for (int p = 0; p < c->world; p++) {
        if (p == c->rank) continue;
        if (send_bytes[p] &&
            check(c, ((fn_send)c->fn[F_SEND])((const char *)send + send_off[p], send_bytes[p], kNcclInt8, p, c->comm, st), "ncclSend"))
            return -1;
        if (recv_bytes[p] &&
            check(c, ((fn_recv)c->fn[F_RECV])((char *)recv + recv_off[p], recv_bytes[p], kNcclInt8, p, c->comm, st), "ncclRecv"))
            return -1;
    }
    return check(c, ((fn_group)c->fn[F_GEND])(), "ncclGroupEnd");
}

int nccl_allgather(NcclComm *c, const void *send, void *recv, size_t bytes_per_rank, cudaStream_t st)
{
    if (c->loop) return loop_allgather(c, send, recv, bytes_per_rank, st);
    return check(c, ((fn_allgather)c->fn[F_ALLGATHER])(send, recv, bytes_per_rank, kNcclInt8, c->comm, st), "ncclAllGather");
}

int nccl_job_begin(NcclComm *c)
{
    if (!c->loop || c->in_job) return 0;
    c->in_job = true;
    return take_turn(c->loop, c->rank);
}

void nccl_job_end(NcclComm *c)
{
    if (!c->loop || !c->in_job) return;
    for (cudaStream_t s : c->streams)
        if (s) cudaStreamSynchronize(s);      // nothing of this rank runs on the device once the turn is released
    c->in_job = false;
    release_turn(c->loop, c->rank);
}

cudaError_t nccl_ipc_export(NcclComm *c, void *ptr, void *handle)
{
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    if (c->loop) {
        memset(handle, 0, sizeof(cudaIpcMemHandle_t));
        memcpy(handle, &ptr, sizeof(ptr));
        return cudaSuccess;
    }
    cudaIpcMemHandle_t h;
    const cudaError_t e = cudaIpcGetMemHandle(&h, ptr);
    memcpy(handle, &h, sizeof(h));
    return e;
}

cudaError_t nccl_ipc_map(NcclComm *c, const void *handle, void **ptr)
{
    if (c->loop) {
        memcpy(ptr, handle, sizeof(*ptr));
        return cudaSuccess;
    }
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, sizeof(h));
    return cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess);
}

cudaError_t nccl_ipc_unmap(NcclComm *c, void *ptr)
{
    return c->loop ? cudaSuccess : cudaIpcCloseMemHandle(ptr);
}

}  // namespace tad

// Registers a loopback group of `world` ranks in this process and writes its 128-byte id.  Passed to tad_init as the
// ncclUniqueId of `world` contexts on one device, it joins them through the loopback instead of NCCL, so that the
// multi-rank paths run on a single GPU (tests).  0 on success.
extern "C" int tad_debug_loopback_id(int world, void *out, size_t bytes)
{
    using namespace tad;
    if (!out || bytes < 128 || world < 2 || world > kLoopRanks) return -1;
    auto g = std::make_shared<Loopback>();
    g->world = world;
    static std::atomic<uint64_t> serial{0};
    g->token = ((uint64_t)std::random_device{}() << 32) ^ ++serial;
    {
        std::lock_guard<std::mutex> lk(g_reg_mu);
        while (g_reg.count(g->token)) g->token++;
        g_reg[g->token] = g;
    }
    memset(out, 0, 128);
    memcpy(out, kLoopMagic, sizeof(kLoopMagic));
    memcpy(static_cast<char *>(out) + 16, &g->token, 8);
    memcpy(static_cast<char *>(out) + 24, &world, 4);
    return 0;
}

// Drops a loopback id from the registry: no further context can join with it.  The ranks that joined keep their group.
// Call it once the ranks are created (or their creation failed), so that an id not every rank joined is not kept for
// the life of the process.  0 on success, also for an id no longer registered.
extern "C" int tad_debug_loopback_release(const void *id, size_t bytes)
{
    using namespace tad;
    if (!id || bytes < 128) return -1;
    if (memcmp(id, kLoopMagic, sizeof(kLoopMagic)) != 0) return -1;
    uint64_t token;
    memcpy(&token, static_cast<const char *>(id) + 16, 8);
    std::lock_guard<std::mutex> lk(g_reg_mu);
    g_reg.erase(token);
    return 0;
}
