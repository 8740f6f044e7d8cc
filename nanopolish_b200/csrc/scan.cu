// scan.cu — the library's exclusive prefix sum over device arrays (record offsets of call-methylation and its TSV rows,
// per-position read and job offsets of variant screening).
//
// Three small launches (per-block sums, a one-block scan of the sums, per-block scan with the block's base) instead of one
// block walking the whole array: 200 000 positions took 0.36 ms per call in the one-block form, ten calls per screening.
#include "nph_internal.cuh"

namespace {

constexpr int kScanBlock = 1024;

// a block's inclusive scan: !APPLY writes the block's total to block_sum, APPLY the exclusive prefix plus the block's base
template <bool APPLY>
__global__ void __launch_bounds__(kScanBlock) nph_scan_block_kernel(const uint64_t* __restrict__ in, uint32_t n, uint64_t* __restrict__ block_sum,
                                                                    uint64_t* __restrict__ out)
{
    __shared__ unsigned long long s[32];
    const uint32_t i = blockIdx.x * kScanBlock + threadIdx.x;
    const unsigned long long v = i < n ? in[i] : 0ull;
    const unsigned long long incl = nph_block_scan_incl(v, s, threadIdx.x);
    if (!APPLY && threadIdx.x == kScanBlock - 1) block_sum[blockIdx.x] = incl;
    if (APPLY && i < n) out[i] = block_sum[blockIdx.x] + incl - v;
}

__global__ void __launch_bounds__(kScanBlock) nph_scan_top_kernel(uint64_t* __restrict__ block_sum, uint32_t n_blocks, uint64_t* __restrict__ total)
{
    __shared__ unsigned long long s[32];
    __shared__ unsigned long long carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < n_blocks; base += kScanBlock) {
        const uint32_t i = base + threadIdx.x;
        const unsigned long long v = i < n_blocks ? block_sum[i] : 0ull;
        const unsigned long long incl = nph_block_scan_incl(v, s, threadIdx.x);
        if (i < n_blocks) block_sum[i] = carry + incl - v;
        __syncthreads();
        if (threadIdx.x == kScanBlock - 1) carry += incl;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = carry;
}

} // namespace

size_t nph_scan_scratch(size_t n) { return (n + kScanBlock - 1) / kScanBlock; }

int nph_scan_exclusive(nph_ctx* ctx, const uint64_t* in, uint32_t n, uint64_t* out, uint64_t* scratch)
{
    const uint32_t nb = (uint32_t)nph_scan_scratch(n);
    // n = 0: only the total (0) is written
    if (nb) nph_scan_block_kernel<false><<<nb, kScanBlock, 0, ctx->stream>>>(in, n, scratch, nullptr);
    nph_scan_top_kernel<<<1, kScanBlock, 0, ctx->stream>>>(scratch, nb, out + n);
    if (nb) nph_scan_block_kernel<true><<<nb, kScanBlock, 0, ctx->stream>>>(in, n, scratch, out);
    NPH_CUDA(ctx, cudaGetLastError());
    return NPH_OK;
}
