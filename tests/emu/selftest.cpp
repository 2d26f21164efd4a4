// TEST INFRASTRUCTURE.  Checks of the CPU emulation itself (tests/emu/include/cuda_runtime.h + emu_runtime.cpp): block
// barriers, warp collectives with full and partial masks, early-exited lanes, atomics, dynamic shared memory, cub stand-ins,
// a one-block "cooperative" kernel whose warps wait for each other through polled flags.  tests/test_emu_device.py compiles
// and runs it; "emu selftest ok" = pass.
#include <cuda_runtime.h>
#include <cooperative_groups.h>
#include <cub/cub.cuh>
#include <numeric>
#define CHECK(c) do { if (!(c)) { std::printf("FAILED line %d: %s\n", __LINE__, #c); std::exit(1); } } while (0)

__global__ void k_reverse(int *data, int n) {                       // __syncthreads + static and dynamic shared memory
    __shared__ int s[256];
    int *dyn = static_cast<int *>(emu::dynamic_smem());
    const int t = threadIdx.x, base = blockIdx.x * blockDim.x;
    if (base + t < n) { s[t] = data[base + t]; dyn[t] = t; }
    __syncthreads();
    const int m = min(int(blockDim.x), n - base);
    if (t < m) data[base + t] = s[m - 1 - t] + dyn[t] - t;
}
__global__ void k_warp(unsigned *out) {                              // collectives, full mask
    const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    unsigned v = lane + 1;
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const unsigned ball = __ballot_sync(0xffffffffu, lane % 3 == 0);
    const unsigned grp = __match_any_sync(0xffffffffu, lane / 8);
    const unsigned mx = __reduce_max_sync(0xffffffffu, lane * 7u % 32u), mn = __reduce_min_sync(0xffffffffu, lane + 5u);
    const unsigned up = __shfl_up_sync(0xffffffffu, lane, 1), dn = __shfl_down_sync(0xffffffffu, lane, 2), bc = __shfl_sync(0xffffffffu, lane * 10u, 3);
    const int smx = __reduce_max_sync(0xffffffffu, lane < 4u ? -7 : (int)lane - 40), smn = __reduce_min_sync(0xffffffffu, (int)lane - 3);
    if (lane == 0) { unsigned *o = out + 8 * warp; o[0] = v; o[1] = ball; o[2] = grp; o[3] = mx; o[4] = mn; out[16 + 2 * warp] = unsigned(smx); out[17 + 2 * warp] = unsigned(smn); }
    if (lane == 5) { unsigned *o = out + 8 * warp; o[5] = up; o[6] = dn; o[7] = bc; }
}
__global__ void k_partial(unsigned *out) {                           // partial masks, lanes that have exited
    const unsigned lane = threadIdx.x & 31u;
    if (lane >= 20) return;
    const unsigned active = __ballot_sync(0x000fffffu, true);
    const unsigned even = __ballot_sync(active, (lane & 1u) == 0);
    if (lane & 1u) return;
    const unsigned sum = __reduce_max_sync(even, lane);
    const int any = __any_sync(even, lane == 18), all = __all_sync(even, lane < 19);
    atomicAdd(&out[0], 1u);
    if (lane == 0) { out[1] = active; out[2] = even; out[3] = sum; out[4] = unsigned(any); out[5] = unsigned(all); }
}
__global__ void k_chain(volatile unsigned *flag, unsigned *order, unsigned *cursor) {     // warps of ONE block hand a token along: polls must yield
    namespace cg = cooperative_groups;
    const unsigned warp = threadIdx.x >> 5, lane = threadIdx.x & 31u, nw = blockDim.x >> 5;
    const unsigned mine = nw - 1 - warp;                              // the last warp goes first
    if (lane == 0) {
        while (*flag != mine) __nanosleep(20);
        order[atomicAdd(cursor, 1u)] = warp;
        *flag = mine + 1;
    }
    __syncwarp();
    cg::this_grid().sync();
    if (threadIdx.x == 0) order[nw] = *flag;
}

int main() {
    {   int n = 1000; std::vector<int> h(n); std::iota(h.begin(), h.end(), 0);
        int *d; cudaMalloc(&d, n * sizeof(int)); cudaMemcpy(d, h.data(), n * sizeof(int), cudaMemcpyHostToDevice);
        EMU_LAUNCH(k_reverse, 4, 256, 256 * sizeof(int), nullptr, d, n);
        cudaMemcpy(h.data(), d, n * sizeof(int), cudaMemcpyDeviceToHost);
        for (int b = 0; b < 4; ++b) { const int base = b * 256, m = std::min(256, n - base); for (int t = 0; t < m; ++t) CHECK(h[base + t] == base + m - 1 - t); }
        cudaFree(d); }
    {   unsigned *d; cudaMalloc(&d, 64 * sizeof(unsigned)); cudaMemset(d, 0, 64 * sizeof(unsigned));
        EMU_LAUNCH(k_warp, 1, 64, 0, nullptr, d);
        for (int w = 0; w < 2; ++w) {
            const unsigned *o = d + 8 * w;
            CHECK(o[0] == 32u * 33u / 2u); CHECK(o[1] == 0x49249249u); CHECK(o[2] == 0x000000ffu); CHECK(o[3] == 31u); CHECK(o[4] == 5u);
            CHECK(o[5] == 4u && o[6] == 7u && o[7] == 30u);
            CHECK(int(d[16 + 2 * w]) == -7 && int(d[17 + 2 * w]) == -3);       // int overloads: signed order
        }
        cudaFree(d); }
    {   unsigned *d; cudaMalloc(&d, 8 * sizeof(unsigned)); cudaMemset(d, 0, 8 * sizeof(unsigned));
        EMU_LAUNCH(k_partial, 1, 32, 0, nullptr, d);
        CHECK(d[0] == 10u); CHECK(d[1] == 0x000fffffu); CHECK(d[2] == 0x00055555u); CHECK(d[3] == 18u); CHECK(d[4] == 1u && d[5] == 1u);
        cudaFree(d); }
    {   unsigned *d; cudaMalloc(&d, 16 * sizeof(unsigned)); cudaMemset(d, 0, 16 * sizeof(unsigned));
        emu::launch(k_chain, dim3(1), dim3(128), 0, (volatile unsigned *)d, d + 2, d + 1);
        CHECK(d[2] == 3u && d[3] == 2u && d[4] == 1u && d[5] == 0u); CHECK(d[6] == 4u);
        cudaFree(d); }
    {   unsigned keys[6] = {5, 1, 5, 3, 1, 2}, vals[6] = {0, 1, 2, 3, 4, 5}, ko[6], vo[6]; size_t bytes = 0; char tmp[256];
        cub::DeviceRadixSort::SortPairs(nullptr, bytes, keys, ko, vals, vo, 6); CHECK(bytes > 0);
        cub::DeviceRadixSort::SortPairs(tmp, bytes, keys, ko, vals, vo, 6);
        const unsigned want_v[6] = {1, 4, 5, 3, 0, 2};                  // stable
        for (int i = 0; i < 6; ++i) CHECK(vo[i] == want_v[i]);
        unsigned in[5] = {3, 0, 2, 2, 1}, out[5];
        cub::DeviceScan::ExclusiveSum(tmp, bytes, in, out, 5);
        CHECK(out[0] == 0 && out[1] == 3 && out[2] == 3 && out[3] == 5 && out[4] == 7); }
    std::puts("emu selftest ok");
    return 0;
}
