// deepterrainrl_b200 -- analysis probe behind cScenarioPoliEval::RecordNNActivation (scenarios/ScenarioPoliEval.cpp:271-296) ->
// cNeuralNet::GetLayerState (learning/NeuralNet.cpp:814-833): the named blob of the deploy net
// (data/policies/dog/nets/dog_mace3_deploy.prototxt) for the policy state of an env's last decision.  The decision kernels keep
// activations in shared memory only, so the probe recomputes the forward pass for ONE env with every blob written to a dump
// buffer -- the pre-activation blobs and the ReLU layers' own top blobs are distinct in that prototxt.  One CTA, plain loops: this
// runs once per recorded gait cycle, not in the step loop.
#include <cuda_runtime.h>

#include <cstring>
#include <string>
#include <vector>

#include "../../include/terrainrl_b200.h"
#include "trl_handle.h"

namespace trl { cudaError_t step_phase_clocks(unsigned long long* out, int reset); }
namespace trl_cg { cudaError_t step_phase_clocks(unsigned long long* out, int reset); }

namespace trl_probe {
using namespace trl;

struct Layout {
    int data, conv0, relu0, conv1, relu1, conv2, relu2, tip0, trelu3, concat0, ip0, hrelu0, h0[4], hr[4], h1[4], output, total;
};
__host__ __device__ inline Layout make_layout(int n_char, int n_frags, int frag) {
    Layout L;
    int o = 0;
    auto take = [&](int n) { int r = o; o += n; return r; };
    L.data = take(200 + n_char);
    L.conv0 = take(16 * 193); L.relu0 = take(16 * 193);
    L.conv1 = take(32 * 190); L.relu1 = take(32 * 190);
    L.conv2 = take(32 * 187); L.relu2 = take(32 * 187);
    L.tip0 = take(64); L.trelu3 = take(64);
    L.concat0 = take(64 + n_char);
    L.ip0 = take(256); L.hrelu0 = take(256);
    for (int k = 0; k < 4; ++k) { L.h0[k] = take(128); L.hr[k] = take(128); L.h1[k] = take(k == 0 ? n_frags : frag); }
    L.output = take(n_frags * (1 + frag));
    L.total = o;
    return L;
}

__device__ void conv_layer(const double* in, int cin, int win, const double* w, const double* b, int cout, int k, double* pre, double* post) {
    const int wout = win - k + 1;
    for (int idx = threadIdx.x; idx < cout * wout; idx += blockDim.x) {
        const int o = idx / wout, t = idx - o * wout;
        double acc = b[o];
        for (int c = 0; c < cin; ++c)
            for (int kk = 0; kk < k; ++kk) acc += w[(o * cin + c) * k + kk] * in[c * win + t + kk];
        pre[idx] = acc; post[idx] = acc > 0.0 ? acc : 0.0;
    }
    __syncthreads();
}
// one output row per warp, lanes stride over the fan-in
__device__ void fc_layer(const double* in, int nin, const double* w, const double* b, int nout, double* pre, double* post) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
    for (int o = warp; o < nout; o += nwarp) {
        double acc = 0.0;
        for (int i = lane; i < nin; i += 32) acc += w[(size_t)o * nin + i] * in[i];
        for (int s = 16; s > 0; s >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, s);
        if (lane == 0) { acc += b[o]; pre[o] = acc; if (post) post[o] = acc > 0.0 ? acc : 0.0; }
    }
    __syncthreads();
}

__global__ void __launch_bounds__(512) trl_layer_probe_kernel(NetWeights W, const double* __restrict__ x, int n_char, int n_frags, int frag, double* dump) {
    const Layout L = make_layout(n_char, n_frags, frag);
    const int n_in = 200 + n_char;
    for (int i = threadIdx.x; i < n_in; i += blockDim.x) dump[L.data + i] = (x[i] + W.in_off[i]) * W.in_scale[i];     // NormalizeInput
    __syncthreads();
    conv_layer(dump + L.data, 1, 200, W.conv0_w, W.conv0_b, 16, 8, dump + L.conv0, dump + L.relu0);
    conv_layer(dump + L.relu0, 16, 193, W.conv1_w, W.conv1_b, 32, 4, dump + L.conv1, dump + L.relu1);
    conv_layer(dump + L.relu1, 32, 190, W.conv2_w, W.conv2_b, 32, 4, dump + L.conv2, dump + L.relu2);
    fc_layer(dump + L.relu2, 32 * 187, W.tip0_w, W.tip0_b, 64, dump + L.tip0, dump + L.trelu3);
    for (int i = threadIdx.x; i < 64 + n_char; i += blockDim.x) dump[L.concat0 + i] = i < 64 ? dump[L.trelu3 + i] : dump[L.data + 200 + (i - 64)];
    __syncthreads();
    fc_layer(dump + L.concat0, 64 + n_char, W.ip0_w, W.ip0_b, 256, dump + L.ip0, dump + L.hrelu0);
    int col = 0;
    for (int k = 0; k < 4; ++k) {
        const int nout = k == 0 ? n_frags : frag;
        fc_layer(dump + L.hrelu0, 256, W.h0_w[k], W.h0_b[k], 128, dump + L.h0[k], dump + L.hr[k]);
        fc_layer(dump + L.hr[k], 128, W.h1_w[k], W.h1_b[k], nout, dump + L.h1[k], nullptr);
        for (int i = threadIdx.x; i < nout; i += blockDim.x) dump[L.output + col + i] = dump[L.h1[k] + i];      // the `output` concat (normalised)
        col += nout;
        __syncthreads();
    }
}
}  // namespace trl_probe

extern "C" int trl_get_layer_state(trl_handle* h, int env, const char* layer_name, double* out, int cap, int* n_out) {
    using namespace trl_probe;
    if (!h) return trl_fail("trl_get_layer_state: null handle");
    if (!h->mc.has_net) return trl_fail("trl_get_layer_state: scene has no policy net");
    if (env < 0 || env >= h->n) return trl_fail("env out of range");
    if (!layer_name || !out) return trl_fail("trl_get_layer_state: null argument");
    const int nc = h->mc.n_char, nf = h->mc.n_frags, fr = h->mc.frag;
    const Layout L = make_layout(nc, nf, fr);
    struct Named { const char* name; int off, size; };
    std::vector<Named> tab = {{"data", L.data, 200 + nc}, {"data_terrain", L.data, 200}, {"data_char", L.data + 200, nc}, {"char_flatten0", L.data + 200, nc},
                              {"terr_conv0", L.conv0, 16 * 193}, {"terr_relu0", L.relu0, 16 * 193}, {"terr_conv1", L.conv1, 32 * 190},
                              {"terr_relu1", L.relu1, 32 * 190}, {"terr_conv2", L.conv2, 32 * 187}, {"terr_relu2", L.relu2, 32 * 187},
                              {"terr_ip0", L.tip0, 64}, {"terr_relu3", L.trelu3, 64}, {"concat0", L.concat0, 64 + nc}, {"ip0", L.ip0, 256}, {"relu0", L.hrelu0, 256},
                              {"output", L.output, nf * (1 + fr)}};
    static const char* heads[4] = {"val", "a0", "a1", "a2"};
    std::vector<std::string> keep;
    keep.reserve(12);
    for (int k = 0; k < 4; ++k) {
        keep.push_back(std::string(heads[k]) + "_ip0"); tab.push_back({keep.back().c_str(), L.h0[k], 128});
        keep.push_back(std::string(heads[k]) + "_relu0"); tab.push_back({keep.back().c_str(), L.hr[k], 128});
        keep.push_back(std::string(heads[k]) + "_ip1"); tab.push_back({keep.back().c_str(), L.h1[k], k == 0 ? nf : fr});
    }
    const Named* hit = nullptr;
    for (const Named& t : tab) if (std::strcmp(t.name, layer_name) == 0) hit = &t;
    if (!hit) return trl_fail(std::string("Can't find layer named ") + layer_name);        // the reference's message (learning/NeuralNet.cpp:830)
    if (!h->probe_dump) {
        if (cudaMalloc((void**)&h->probe_dump, (size_t)L.total * 8) != cudaSuccess) return trl_fail("trl_get_layer_state: out of device memory");
        h->allocs.push_back(h->probe_dump);
    }
    TRL_LAUNCH(trl_layer_probe_kernel, 1, 512, 0, h->stream, env_policy(h, env), (const double*)(h->B.poli_state + (size_t)env * h->B.S), nc, nf, fr, h->probe_dump);
    h->launches += 1;
    if (cudaGetLastError() != cudaSuccess || cudaStreamSynchronize(h->stream) != cudaSuccess) return trl_fail("trl_get_layer_state: probe kernel failed");
    const int n = std::min(hit->size, cap);
    if (cudaMemcpy(out, h->probe_dump + hit->off, (size_t)n * 8, cudaMemcpyDeviceToHost) != cudaSuccess) return trl_fail("trl_get_layer_state: copy failed");
    if (n_out) *n_out = hit->size;
    return 0;
}

// Per-phase clock64() sums of the env-step kernel (both builds: main and catch-up launches), in a TRL_PHASE_CLOCKS=1 build only.
// out[0..n-2] = cycles summed over warps per phase, out[n-1] = env-steps (physics halves) counted; reset zeroes the counters.
extern "C" int trl_debug_step_phases(trl_handle* h, unsigned long long* out, int n, int reset) {
    constexpr int kSlots = 10;
    if (!h || !out || n != kSlots) return trl_fail("trl_debug_step_phases: null handle / output, or n != 10");
    if (cudaStreamSynchronize(h->stream) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) return trl_fail("trl_debug_step_phases: sync failed");
    unsigned long long a[kSlots], b[kSlots];
    if (trl::step_phase_clocks(a, reset) != cudaSuccess || trl_cg::step_phase_clocks(b, reset) != cudaSuccess)
        return trl_fail("trl_debug_step_phases: the library was built without -DTRL_PHASE_CLOCKS=1 (TRL_VARIANT=phase_clocks)");
    for (int k = 0; k < kSlots; ++k) out[k] = a[k] + b[k];
    return 0;
}
