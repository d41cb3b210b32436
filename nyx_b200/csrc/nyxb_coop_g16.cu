// nyxb_coop_g16.cu — instantiation of the lane-cooperative kernel for 16 lanes per trajectory group
#include "nyxb_coop_kernel.cuh"

cudaError_t nyxb_launch_coop_g16(const DevSetup* S, const DevCoop* Cp, size_t n, const double* state, const double* consts,
                                 const long long* epoch0, long long end_epoch, long long* step_io, double* out_state,
                                 long long* out_epoch, nyxb_details* out_details, int* out_status, const DevSink* sink,
                                 cudaStream_t stream) {
    return nyxb_launch_coop_g<16>(S, Cp, n, state, consts, epoch0, end_epoch, step_io, out_state, out_epoch, out_details,
                                  out_status, sink, stream);
}
