// l2_tma_probe.cu -- L2 -> shared-memory bandwidth of TMA tile loads, the operand feed of k_conv_tc.
//
// One CTA per SM.  One thread keeps a ring of S shared-memory stages full: it waits for a stage's mbarrier, re-arms it and
// loads the next [rows x 64 bf16] box (128-byte rows, 128B swizzle: the A / B tiles of a BK = 64 K-block) from a 16 MB tensor
// that stays resident in L2.  Prints the aggregate bytes/s per (box rows, stages).
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o l2_tma_probe tools/l2_tma_probe.cu
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

__global__ void __launch_bounds__(32, 1) k_probe(const __grid_constant__ CUtensorMap tm, int box_rows, int nboxes, int stages, int iters) {
    extern __shared__ unsigned char smem_raw[];
    const uint32_t base = ((uint32_t)__cvta_generic_to_shared(smem_raw) + 1023u) & ~1023u;
    const uint32_t box_bytes = (uint32_t)box_rows * 128u;
    const uint32_t bars = base + (uint32_t)stages * box_bytes;
    if (threadIdx.x != 0) return;
    for (int s = 0; s < stages; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bars + 8u * s));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    uint32_t box = (uint32_t)blockIdx.x * 7919u;
    for (int i = 0; i < iters + stages; ++i) {
        const int s = i % stages;
        const uint32_t bar = bars + 8u * s;
        if (i >= stages) {   // the load issued `stages` iterations ago into this stage has landed
            const uint32_t parity = (uint32_t)((i / stages - 1) & 1);
            uint32_t ok = 0;
            while (!ok)
                asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}"
                             : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
        }
        if (i >= iters) continue;
        box = (box + 131u) % (uint32_t)nboxes;
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(box_bytes) : "memory");
        asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                     ::"r"(base + (uint32_t)s * box_bytes), "l"(&tm), "r"(bar), "r"(0), "r"((int)(box * (uint32_t)box_rows)) : "memory");
    }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int main() {
    int dev = 0, sms = 0, clk = 0;
    CK(cudaGetDevice(&dev));
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, dev));
    CK(cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, dev));
    const size_t bytes = 16u << 20, rows = bytes / 128;
    void *buf = nullptr;
    CK(cudaMalloc(&buf, bytes));
    CK(cudaMemset(buf, 1, bytes));
    void *fp = nullptr;
    cudaDriverEntryPointQueryResult q;
    CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q));
    EncodeTiledFn enc = reinterpret_cast<EncodeTiledFn>(fp);
    CK(cudaFuncSetAttribute(k_probe, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    printf("device %s, %d SMs, max SM clock %d MHz; 16 MB L2-resident source, one CTA per SM\n", prop.name, sms, clk / 1000);
    printf("%9s %7s %10s %12s\n", "box_rows", "stages", "KB/SM", "GB/s");
    const int box_rows_list[] = {128, 256};
    const int stages_list[] = {2, 3, 4, 5, 6, 8, 12};
    for (int box_rows : box_rows_list) {
        CUtensorMap tm;
        cuuint64_t dims[2] = {64, (cuuint64_t)rows};
        cuuint64_t strides[1] = {128};
        cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
        cuuint32_t es[2] = {1, 1};
        if (enc(&tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, buf, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) {
            fprintf(stderr, "cuTensorMapEncodeTiled failed\n");
            return 1;
        }
        const int nboxes = (int)(rows / box_rows);
        for (int stages : stages_list) {
            const size_t smem = 1024 + (size_t)stages * box_rows * 128 + 8 * stages;
            if (smem > 227 * 1024) continue;
            const int iters = (int)((4096LL * 128) / box_rows);   // 64 MB per SM per launch
            k_probe<<<sms, 32, smem>>>(tm, box_rows, nboxes, stages, iters / 8);   // warm-up (and L2 fill)
            CK(cudaGetLastError());
            CK(cudaDeviceSynchronize());
            cudaEvent_t e0, e1;
            CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
            std::vector<float> ms;
            for (int rep = 0; rep < 5; ++rep) {
                CK(cudaEventRecord(e0));
                k_probe<<<sms, 32, smem>>>(tm, box_rows, nboxes, stages, iters);
                CK(cudaEventRecord(e1));
                CK(cudaEventSynchronize(e1));
                float t = 0.f;
                CK(cudaEventElapsedTime(&t, e0, e1));
                ms.push_back(t);
            }
            std::sort(ms.begin(), ms.end());
            const double moved = (double)sms * iters * box_rows * 128.0;
            printf("%9d %7d %10d %12.0f\n", box_rows, stages, stages * box_rows * 128 / 1024, moved / (ms[2] * 1e-3) / 1e9);
            CK(cudaEventDestroy(e0)); CK(cudaEventDestroy(e1));
        }
    }
    CK(cudaFree(buf));
    return 0;
}
