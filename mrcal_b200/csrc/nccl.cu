// Multi-GPU plumbing: one process per GPU, one NCCL communicator, one
// all-reduce (fp64 sum) of the reduced normal equations per iteration
// (solver.cu). NCCL is loaded at run time with dlopen() so that the library has
// no link-time dependency on it: single-GPU use needs no NCCL at all. The
// unique id travels between processes by whatever the host side has
// (torch.distributed in mrcal_b200/distributed.py).
#include <dlfcn.h>

#include "comm.h"
#include "problem_impl.h"

namespace mb200 {

struct NcclUniqueId { char internal[128]; };
typedef void* ncclComm_t;
typedef int (*fn_GetUniqueId)(NcclUniqueId*);
typedef int (*fn_CommInitRank)(ncclComm_t*, int, NcclUniqueId, int);
typedef int (*fn_AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t);
typedef int (*fn_CommDestroy)(ncclComm_t);
typedef const char* (*fn_GetErrorString)(int);

static struct
{
    void* handle = nullptr;
    fn_GetUniqueId GetUniqueId = nullptr;
    fn_CommInitRank CommInitRank = nullptr;
    fn_AllReduce AllReduce = nullptr;
    fn_CommDestroy CommDestroy = nullptr;
    fn_GetErrorString GetErrorString = nullptr;
    ncclComm_t comm = nullptr;
    int rank = 0, nranks = 1;
} g_nccl;

static bool load_nccl()
{
    if(g_nccl.handle) return true;
    const char* env = getenv("MRCAL_B200_NCCL_LIB");
    const char* candidates[] = {env, "libnccl.so.2", "libnccl.so"};
    for(const char* c : candidates)
    {
        if(c == nullptr || !*c) continue;
        g_nccl.handle = dlopen(c, RTLD_NOW | RTLD_GLOBAL);
        if(g_nccl.handle) break;
    }
    if(!g_nccl.handle)
    {
        set_error("could not load NCCL (set MRCAL_B200_NCCL_LIB to the path of libnccl.so.2): %s", dlerror());
        return false;
    }
    g_nccl.GetUniqueId    = (fn_GetUniqueId)dlsym(g_nccl.handle, "ncclGetUniqueId");
    g_nccl.CommInitRank   = (fn_CommInitRank)dlsym(g_nccl.handle, "ncclCommInitRank");
    g_nccl.AllReduce      = (fn_AllReduce)dlsym(g_nccl.handle, "ncclAllReduce");
    g_nccl.CommDestroy    = (fn_CommDestroy)dlsym(g_nccl.handle, "ncclCommDestroy");
    g_nccl.GetErrorString = (fn_GetErrorString)dlsym(g_nccl.handle, "ncclGetErrorString");
    if(!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.AllReduce || !g_nccl.CommDestroy)
    {
        set_error("the NCCL library lacks a required symbol");
        return false;
    }
    return true;
}

static long g_collectives = 0;   // all-reduce calls issued (a figure for DESIGN.md / bench.py)
long comm_collective_count() { return g_collectives; }
bool comm_active() { return g_nccl.comm != nullptr && g_nccl.nranks > 1; }
int  comm_rank() { return g_nccl.rank; }
int  comm_size() { return g_nccl.nranks; }

bool comm_allreduce_sum(double* d_buf, size_t count, cudaStream_t s)
{
    if(!comm_active()) return true;
    g_collectives++;
    const int rc = g_nccl.AllReduce(d_buf, d_buf, count, /*ncclFloat64*/ 8, /*ncclSum*/ 0, g_nccl.comm, s);
    if(rc != 0)
    {
        set_error("ncclAllReduce failed: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "?");
        return false;
    }
    return true;
}

bool comm_allreduce_max_int(int* d_buf, size_t count, cudaStream_t s)
{
    if(!comm_active()) return true;
    g_collectives++;
    const int rc = g_nccl.AllReduce(d_buf, d_buf, count, /*ncclInt32*/ 2, /*ncclMax*/ 2, g_nccl.comm, s);
    if(rc != 0)
    {
        set_error("ncclAllReduce(max) failed: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "?");
        return false;
    }
    return true;
}

}  // namespace mb200
using namespace mb200;

extern "C" bool mrcal_b200_nccl_get_unique_id(void* id128)
{
    if(!load_nccl()) return false;
    NcclUniqueId id;
    const int rc = g_nccl.GetUniqueId(&id);
    if(rc != 0) { set_error("ncclGetUniqueId failed: %d", rc); return false; }
    memcpy(id128, &id, 128);
    return true;
}

extern "C" bool mrcal_b200_nccl_comm_init(const void* id128, int rank, int nranks, int device)
{
    if(!load_nccl()) return false;
    if(g_nccl.comm) { set_error("NCCL communicator already initialised"); return false; }
    MB200_CUDA_CHECK(cudaSetDevice(device));
    NcclUniqueId id;
    memcpy(&id, id128, 128);
    const int rc = g_nccl.CommInitRank(&g_nccl.comm, nranks, id, rank);
    if(rc != 0)
    {
        set_error("ncclCommInitRank failed: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "?");
        g_nccl.comm = nullptr;
        return false;
    }
    g_nccl.rank = rank;
    g_nccl.nranks = nranks;
    return true;
}

// Timing aid (not on any product path): device milliseconds per all-reduce (sum) of `count` doubles, back to back
extern "C" double mrcal_b200_debug_time_allreduce(size_t count, int reps)
{
    if(!comm_active()) { set_error("no communicator"); return -1.; }
    double* buf = nullptr;
    cudaStream_t s;
    if(cudaMalloc(&buf, count * sizeof(double)) != cudaSuccess || cudaMemset(buf, 0, count * sizeof(double)) != cudaSuccess ||
       cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) != cudaSuccess) return -1.;
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    for(int r = -3; r < reps; r++)
    {
        if(r == 0) cudaEventRecord(e0, s);
        if(!comm_allreduce_sum(buf, count, s)) return -1.;
    }
    cudaEventRecord(e1, s);
    cudaEventSynchronize(e1);
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e0, e1);
    cudaEventDestroy(e0); cudaEventDestroy(e1); cudaStreamDestroy(s); cudaFree(buf);
    return ms / reps;
}

extern "C" void mrcal_b200_nccl_comm_destroy(void)
{
    if(g_nccl.comm) { g_nccl.CommDestroy(g_nccl.comm); g_nccl.comm = nullptr; }
    g_nccl.rank = 0;
    g_nccl.nranks = 1;
}

extern "C" bool mrcal_b200_problem_set_sharding(mrcal_b200_problem_t* P, int frame_offset, int Nframes_global,
                                                int point_offset, int Npoints_global)
{
    if(P->dp.Ntri > 0) { set_error("sharded solves with triangulated points are not supported"); return false; }
    P->sharded = true;
    P->dp.reg_owner = comm_rank() == 0;
    P->frame_offset = frame_offset; P->Nframes_global = Nframes_global;
    P->point_offset = point_offset; P->Npoints_global = Npoints_global;
    return true;
}
