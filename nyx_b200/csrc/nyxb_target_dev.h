// nyxb_target_dev.h — the device buffers of one nyxb_target_batch call and the launchers of nyxb_target.cu.
#pragma once
#include <cuda_runtime.h>

#include "../../include/nyxb.h"

struct TgtDev {
    size_t n;                 // problems
    // per problem, stride n
    const double* consts;     // [4][n]
    double* start;            // [9][n] the state at the correction epoch
    long long* epoch_c;       // [n]
    double* xi;               // [6][n] the iterated state
    double* total;            // [V][n]
    double* err;              // [O][n]
    double* prev_norm;        // [n]
    double* achieved;         // [9][n]
    double* corrected;        // [9][n]
    int* iters;               // [n]
    int* status;              // [n] the warn flags while a problem iterates, then its status
    int* idx;                 // [n] the active problems (identity after init)
    int* flag;                // [n] 1 = goes on, by position in the active list
    // propagation slab, stride M = A (V + 1)
    double* l_state;          // [9][M]
    double* l_consts;         // [4][M]
    long long* l_epoch;       // [M]
    double* o_state;          // [9][M]
    int* o_status;            // [M]
};

cudaError_t nyxb_tgt_launch_init(const TgtDev& t, const nyxb_target_config& cfg, const double* pre_state, const long long* pre_epoch,
                                 const int* pre_status, cudaStream_t st);
cudaError_t nyxb_tgt_launch_stage(const TgtDev& t, const nyxb_target_config& cfg, int A, const int* idx, cudaStream_t st);
cudaError_t nyxb_tgt_launch_update(const TgtDev& t, const nyxb_target_config& cfg, double mu, int A, const int* idx, cudaStream_t st);
cudaError_t nyxb_tgt_launch_finish(const TgtDev& t, const nyxb_target_config& cfg, cudaStream_t st);
cudaError_t nyxb_tgt_compact(void* temp, size_t* temp_bytes, const int* in, const int* flag, int* out, int* count, int A, cudaStream_t st);
