// Internal: the cross-rank collectives of sharded solves (nccl.cu). Without a communicator of more than one rank they
// do nothing and succeed
#pragma once
#include <cstddef>
#include <cuda_runtime.h>

namespace mb200 {

bool comm_active();
int  comm_rank();
int  comm_size();
long comm_collective_count();   // all-reduce calls issued so far
bool comm_allreduce_sum(double* d_buf, size_t count, cudaStream_t s);
bool comm_allreduce_max_int(int* d_buf, size_t count, cudaStream_t s);

}  // namespace mb200
