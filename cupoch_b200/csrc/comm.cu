// comm.cu -- the one exchange of the sharded ICP: 32 doubles per iteration.
//   kind NCCL: ncclAllReduce, NCCL bound at run time (dlopen) so the library loads on hosts without
//              NCCL and shares the process's libnccl.so.2 (torch's) when one is already loaded;
//   kind P2P : every rank owns a mailbox in its own HBM, mapped into every peer by CUDA IPC.  The last
//              block of icp_reduce_kernel stores its 32 partial sums straight into all peers' mailboxes
//              over NVLink, raises a flag, waits for the peers' flags and adds the slots in rank order --
//              the collective is fused into the kernel (no NCCL launch, no separate finalize launch) and
//              the total is bit-identical on every rank.
#include <dlfcn.h>
#include <string.h>

#include <memory>

#include "cphb_internal.cuh"

typedef struct { char internal[128]; } nccl_uid;
typedef void *nccl_comm_t;
typedef int (*fn_get_uid)(nccl_uid *);
typedef int (*fn_init_rank)(nccl_comm_t *, int, nccl_uid, int);
typedef int (*fn_destroy)(nccl_comm_t);
typedef int (*fn_allreduce)(const void *, void *, size_t, int, int, nccl_comm_t, cudaStream_t);
typedef const char *(*fn_errstr)(int);

static struct {
    void *h;
    fn_get_uid get_uid;
    fn_init_rank init_rank;
    fn_destroy destroy;
    fn_allreduce allreduce;
    fn_errstr errstr;
} g_nccl;

static int nccl_load() {
    if (g_nccl.h) return CPHB_OK;
    const char *names[] = {"libnccl.so.2", "libnccl.so", nullptr};
    void *h = nullptr;
    for (int i = 0; names[i] && !h; ++i) h = dlopen(names[i], RTLD_NOW | RTLD_GLOBAL);
    if (!h) {
        cphb_set_error("NCCL not found (dlopen libnccl.so.2): %s", dlerror());
        return CPHB_ERR_NCCL;
    }
    g_nccl.get_uid = (fn_get_uid)dlsym(h, "ncclGetUniqueId");
    g_nccl.init_rank = (fn_init_rank)dlsym(h, "ncclCommInitRank");
    g_nccl.destroy = (fn_destroy)dlsym(h, "ncclCommDestroy");
    g_nccl.allreduce = (fn_allreduce)dlsym(h, "ncclAllReduce");
    g_nccl.errstr = (fn_errstr)dlsym(h, "ncclGetErrorString");
    if (!g_nccl.get_uid || !g_nccl.init_rank || !g_nccl.destroy || !g_nccl.allreduce) {
        cphb_set_error("NCCL symbols missing");
        return CPHB_ERR_NCCL;
    }
    g_nccl.h = h;
    return CPHB_OK;
}
#define NCCL_TRY(x)                                                                          \
    do {                                                                                     \
        int r__ = (x);                                                                       \
        if (r__ != 0) {                                                                      \
            cphb_set_error("%s: %s", #x, g_nccl.errstr ? g_nccl.errstr(r__) : "nccl error"); \
            return CPHB_ERR_NCCL;                                                            \
        }                                                                                    \
    } while (0)

extern "C" int cphb_nccl_unique_id(char h_id[128]) {
    int rc = nccl_load();
    if (rc) return rc;
    nccl_uid u;
    NCCL_TRY(g_nccl.get_uid(&u));
    memcpy(h_id, u.internal, 128);
    return CPHB_OK;
}

int cphb_nccl_allreduce_f64(void *comm, const double *send, double *recv, size_t count, cudaStream_t s) {
    int rc = nccl_load();
    if (rc) return rc;
    // ncclFloat64 = 8, ncclSum = 0 (nccl.h)
    NCCL_TRY(g_nccl.allreduce(send, recv, count, 8, 0, (nccl_comm_t)comm, s));
    return CPHB_OK;
}

// ---------------------------------------------------------------------------
// cphb_comm
// ---------------------------------------------------------------------------
extern "C" int cphb_comm_nccl_create(const char h_id[128], int world_size, int rank, cphb_comm **out) {
    int rc = nccl_load();
    if (rc) return rc;
    nccl_uid u;
    memcpy(u.internal, h_id, 128);
    nccl_comm_t c = nullptr;
    NCCL_TRY(g_nccl.init_rank(&c, world_size, u, rank));
    cphb_comm *cm = new cphb_comm();
    cm->kind = CPHB_COMM_NCCL;
    cm->rank = rank;
    cm->world = world_size;
    cm->nccl = c;
    *out = cm;
    return CPHB_OK;
}

extern "C" int cphb_comm_p2p_create(int world_size, int rank, char h_handle[64], cphb_comm **out) {
    if (world_size < 1 || world_size > CPHB_P2P_MAX_WORLD || rank < 0 || rank >= world_size) {
        cphb_set_error("cphb_comm_p2p_create: world %d / rank %d unsupported (max %d)", world_size, rank, CPHB_P2P_MAX_WORLD);
        return CPHB_ERR_INVALID;
    }
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    std::unique_ptr<cphb_comm> cm(new cphb_comm());
    cm->kind = CPHB_COMM_P2P;
    cm->rank = rank;
    cm->world = world_size;
    CPHB_CUDA(cudaMalloc(&cm->box_local, CPHB_P2P_ALLOC_BYTES));  // IPC needs cudaMalloc memory, not the async pool
    CPHB_CUDA(cudaMemset(cm->box_local, 0, CPHB_P2P_ALLOC_BYTES));
    CPHB_CUDA(cudaDeviceSynchronize());
    cudaIpcMemHandle_t h;
    CPHB_CUDA(cudaIpcGetMemHandle(&h, cm->box_local));
    memcpy(h_handle, &h, 64);
    *out = cm.release();
    return CPHB_OK;
}

extern "C" int cphb_comm_p2p_connect(cphb_comm *cm, const char *h_handles) {
    if (!cm || cm->kind != CPHB_COMM_P2P || !h_handles) {
        cphb_set_error("cphb_comm_p2p_connect: bad argument");
        return CPHB_ERR_INVALID;
    }
    for (int q = 0; q < cm->world; ++q) {
        if (q == cm->rank) {
            cm->view.box[q] = (char *)cm->box_local;
            continue;
        }
        cudaIpcMemHandle_t h;
        memcpy(&h, h_handles + 64 * (size_t)q, 64);
        void *p = nullptr;
        CPHB_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
        cm->view.box[q] = (char *)p;
    }
    cm->view.rank = cm->rank;
    cm->view.world = cm->world;
    cm->connected = 1;
    return CPHB_OK;
}

cphb_comm::~cphb_comm() {
    if (kind == CPHB_COMM_NCCL && nccl) {
        if (nccl_load() == CPHB_OK) g_nccl.destroy((nccl_comm_t)nccl);
    } else if (kind == CPHB_COMM_P2P) {
        cudaDeviceSynchronize();
        for (int q = 0; q < world; ++q)
            if (q != rank && view.box[q]) cudaIpcCloseMemHandle(view.box[q]);
        if (box_local) cudaFree(box_local);
    }
}

extern "C" int cphb_comm_destroy(cphb_comm *cm) {
    delete cm;
    return CPHB_OK;
}

// stand-alone exchange (count <= 32 doubles, in place): used for the global source size and by tests
__global__ void p2p_allreduce_kernel(P2pView v, double *buf, int count) {
    const int c = threadIdx.x;
    double t = (c < count) ? buf[c] : 0.0;
    t = p2p_exchange_sum(v, t);
    if (c < count) buf[c] = t;
}

extern "C" int cphb_comm_allreduce_f64(cphb_comm *cm, double *buf, int count, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!cm || count < 0 || count > 32) {
        cphb_set_error("cphb_comm_allreduce_f64: bad argument");
        return CPHB_ERR_INVALID;
    }
    if (cm->kind == CPHB_COMM_NCCL) return cphb_nccl_allreduce_f64(cm->nccl, buf, buf, (size_t)count, s);
    if (!cm->connected) {
        cphb_set_error("cphb_comm_allreduce_f64: p2p comm not connected");
        return CPHB_ERR_INVALID;
    }
    CPHB_LAUNCH(p2p_allreduce_kernel, 1, 32, 0, s, cm->view, buf, count);
    CPHB_CHECK_LAUNCH();
    return CPHB_OK;
}
