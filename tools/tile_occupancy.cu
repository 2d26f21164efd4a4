// Resident CTAs and warps per SM of the island-tile kernels, from the occupancy API at the block size and dynamic
// shared memory the world launches them with (b2d_create).  Built and run by tools/tile_residency.py.
#include "../edyn_b200/csrc/b2d_kernels.cuh"
#include <cstdio>

using namespace b2d;

template <typename K>
static int report(const char *name, K kernel, int threads, size_t smem) {
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return 1;
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem) != cudaSuccess) return 1;
    cudaFuncAttributes a;
    if (cudaFuncGetAttributes(&a, kernel) != cudaSuccess) return 1;
    printf("%s: %d threads, %zu B dynamic + %zu B static smem, %d registers, %zu B local: %d CTAs = %d warps per SM\n",
           name, threads, smem, (size_t)a.sharedSizeBytes, a.numRegs, (size_t)a.localSizeBytes, per_sm, per_sm * threads / 32);
    return 0;
}

int main() {
    int rc = report("k_island_tiles", k_island_tiles, TILE_CAP, TILE_FUSED_SMEM);
    rc = rc ? rc : report("k_island_tiles_2p", k_island_tiles_2p, TILE_CAP, TILE_FUSED_SMEM_2P);
    if (rc) fprintf(stderr, "tile_occupancy: %s\n", cudaGetErrorString(cudaGetLastError()));
    return rc;
}
