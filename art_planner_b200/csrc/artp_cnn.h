// art_planner_b200/csrc/artp_cnn.h -- host interface of the motion-cost network (artp_cnn.cu) used by artp_capi.cu.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <string>

namespace artp_cnn {
// The two architectures (values of ARTP_COST_NET_LIGHT / ARTP_COST_NET_FULL); the blob length tells them apart.
constexpr int kNetLight = 0, kNetFull = 1, kNumNetworks = 2;
struct State;
size_t blob_floats(int network);   // 0 for an unknown network
State* create(int device, int sm_count);
void destroy(State* s);
int set_weights(State* s, const float* host_blob, size_t n, cudaStream_t st, std::string& err);
int update_features(State* s, const float* d_layer, int rows, int cols, int pitch, double res, double cx, double cy,
                    cudaStream_t st, int use_reference_conv15, std::string& err);
int motion_cost(State* s, const float* d_edges, size_t n, float* d_cost3, cudaStream_t st, std::string& err);
int copy_features(State* s, float* host_out, size_t n_floats, std::string& err);
void feature_shape(const State* s, int* hf, int* wf);
int network(const State* s);       // the loaded network, -1 before any weights
bool has_features(const State* s);
bool has_weights(const State* s);
void last_times(const State* s, float* ms3);
}  // namespace artp_cnn
