// k4_ptx.cuh -- the sm_90 PTX primitives of the decoder and the marchers other than warpgroup MMAs (k4_wgmma.cuh):
// mbarriers, TMA bulk / tensor copies, cp.async, named barriers, register reallocation, programmatic dependent launch,
// mma.sync / ldmatrix, fp16x2 conversions and two single-use instructions.  One definition each; every inline PTX
// statement of the library is here or in k4_wgmma.cuh.
//
// Shared-memory operands are passed as generic pointers into shared memory and converted with smem_u32.  The fp16x2
// conversions take (lo, hi) and return the packed word with lo in the low half; the names say whether they saturate.
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarriers ----
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" :: "r"(smem_u32(bar)), "r"(count));
}
// makes the mbarrier.init of this thread visible to the other threads and to the async proxy (TMA)
__device__ __forceinline__ void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" :: "r"(smem_u32(bar)) : "memory");
}
// arrive and add `bytes` to the transaction count the current phase waits for
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok = 0;
    while (!ok) {
        asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n"
                     : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    }
}

// ---- TMA: global -> shared copies that complete on an mbarrier ----
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n"
                 :: "r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// the box of a tensor map at coordinates (c0, c1[, c2]), innermost first; out-of-range elements arrive as zeros.
// tmap: the generic address of the CUtensorMap, a __grid_constant__ kernel parameter.
__device__ __forceinline__ void tensor_g2s_2d(void* dst, uint64_t tmap, uint64_t* bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];\n"
                 :: "r"(smem_u32(dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tensor_g2s_3d(void* dst, uint64_t tmap, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];\n"
                 :: "r"(smem_u32(dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
// orders this thread's generic-proxy shared-memory writes before later async-proxy (TMA, wgmma) accesses
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }

// ---- cp.async: 16 bytes, of which the first src_bytes are read and the rest zero filled ----
__device__ __forceinline__ void cp_async16(void* dst, const void* src, int src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" :: "r"(smem_u32(dst)), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
// wait until at most N of this thread's committed groups are pending
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" :: "n"(N) : "memory"); }

// ---- named barriers and register reallocation ----
// named barrier `id` over the 128 threads of a warpgroup (0 is __syncthreads), and its form that also ORs a predicate
// over them
__device__ __forceinline__ void named_bar(int id) { asm volatile("bar.sync %0, 128;\n" :: "r"(id) : "memory"); }
__device__ __forceinline__ bool named_bar_or(int id, bool pred) {
    uint32_t r;
    asm volatile("{\n.reg .pred p, q;\nsetp.ne.u32 p, %2, 0;\nbarrier.cta.red.or.pred q, %1, 128, p;\nselp.u32 %0, 1, 0, q;\n}\n"
                 : "=r"(r) : "r"(id), "r"((uint32_t)pred) : "memory");
    return r != 0;
}
// a warpgroup's per-thread register budget, raised or lowered to N
template <int N> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" :: "n"(N)); }
template <int N> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" :: "n"(N)); }

// ---- programmatic dependent launch ----
// Wait for the preceding kernel's results, then let the next kernel launch.  Nothing produced by an earlier kernel may
// be touched before this call; releasing the dependents only after the wait keeps at most two kernels in flight.
__device__ __forceinline__ void pdl_wait_and_release() {
    asm volatile("griddepcontrol.wait;\n" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;\n" ::: "memory");
}

// ---- warp-level MMA: mma.sync m16n8k16 (fp16 operands, fp32 accumulate) and its ldmatrix operand loads ----
__device__ __forceinline__ void mma_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x2(uint32_t addr, uint32_t& r0, uint32_t& r1) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0,%1}, [%2];\n"
                 : "=r"(r0), "=r"(r1) : "r"(addr));
}

// ---- fp32 pair -> fp16x2, round to nearest ----
// not saturating: beyond +-65504 a value becomes +-inf
__device__ __forceinline__ uint32_t h2_rn(float lo, float hi) {
    __half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&h);
}
// saturating: beyond the fp16 range a value becomes +-65504, never inf (a clamped operand degrades gracefully, an inf
// poisons every later result)
__device__ __forceinline__ uint32_t h2_sat(float lo, float hi) {
    uint32_t d;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;\n" : "=r"(d) : "f"(hi), "f"(lo));
    return d;
}
// ReLU, then saturating
__device__ __forceinline__ uint32_t h2_relu_sat(float lo, float hi) {
    uint32_t d;
    asm("cvt.rn.relu.satfinite.f16x2.f32 %0, %1, %2;\n" : "=r"(d) : "f"(hi), "f"(lo));
    return d;
}
// not saturating hi / lo split of a pair: hi = fp16(x), lo = fp16(x - hi)
__device__ __forceinline__ void split_h2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
    __half2 h = __floats2half2_rn(x0, x1);
    float2 hf = __half22float2(h);
    __half2 l = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
    hi = *reinterpret_cast<uint32_t*>(&h);
    lo = *reinterpret_cast<uint32_t*>(&l);
}

// ---- single instructions ----
// 2^x, approximate, denormals flushed to zero
__device__ __forceinline__ float ex2_approx_ftz(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;\n" : "=f"(y) : "f"(x));
    return y;
}
// the SM's 64-bit cycle counter; volatile with a memory clobber, so it is not moved across the code it times
__device__ __forceinline__ unsigned long long clock64_now() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%clock64;\n" : "=l"(t) :: "memory");
    return t;
}
