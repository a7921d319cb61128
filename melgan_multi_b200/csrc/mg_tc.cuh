// sm_90a tensor-core plumbing: mbarrier, 1-D bulk TMA, warpgroup MMA (wgmma) with shared-memory matrix descriptors
// (no-swizzle, K-major) and fp32 accumulators in registers.
//
// Layout convention used everywhere in this engine ("row-linear K-major, no swizzle"):
//   an operand tile of R rows (M or N index) by K bf16 elements is stored as K/8 "k-panels";
//   panel kp holds, for every row r, the 8 consecutive K elements [8*kp, 8*kp+8) as one 16-byte unit at
//       panel_base(kp) + r * 16.
//   In wgmma terms the core matrix is 8 rows x 16 B = 128 contiguous bytes, the stride between 8-row
//   groups (SBO) is 128 B -- i.e. rows are simply 16 B apart -- and the stride between the two k-panels
//   one K = 16 MMA consumes (LBO) is the panel pitch.  Because rows are linear, a conv tap that shifts the
//   operand by d rows is just "start address + 16*d": no swizzle phase to respect, any d is legal.
//
// Accumulators: one wgmma.m64nNk16 is issued by a whole warpgroup (128 threads) and leaves its 64 x N fp32 result in
// the registers of that warpgroup.  Thread t (warp w = t / 32 of the group, lane l) holds, for every 8-column block k,
//     d[4k + 2h + e] = D[16 w + l / 4 + 8 h][8 k + 2 (l % 4) + e]        (h, e in {0, 1})
// frag_row() / frag_col() below name those coordinates.
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

namespace mg {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier ------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: returns false (and lets the caller raise the status word and carry on) instead of hanging the GPU if the
// producer never arrives.
__device__ __forceinline__ bool mbar_wait(uint64_t *bar, uint32_t parity, uint32_t max_spins = 1u << 24) {
    for (uint32_t i = 0; i < max_spins; ++i)
        if (mbar_try_wait(bar, parity)) return true;
    return false;
}

// ---- thread-block clusters ------------------------------------------------------------------------
// shared::cluster address of the object at shared::cta address `addr` in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t mapa(uint32_t addr, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
    return r;
}
// arrive on the mbarrier `bar` (own shared::cta address) of CTA `rank`, for a consumer that frees a buffer once its MMAs
// (async proxy, completed by wgmma_wait) have read it.  No cluster-scope release: that fence would wait on the whole GPU
// memory system; data for another CTA travels by bulk copy (bulk_s2s_cluster), which completes on the reader's mbarrier.
__device__ __forceinline__ void mbar_arrive_remote(uint64_t *bar, uint32_t rank) {
    asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(mapa(smem_u32(bar), rank)) : "memory");
}
// every thread of every CTA of the cluster; orders shared-memory accesses across the cluster (not bounded: used only
// after barrier initialisation and before exit, where every CTA arrives on every path)
__device__ __forceinline__ void cluster_sync() {
    asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}

// ---- 1-D bulk async copy (TMA, no tensor map): global -> shared, completes on an mbarrier -------
__device__ __forceinline__ void bulk_g2s(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// the same copy landing at the same shared-memory offset of every CTA in `cta_mask` (one L2 read), each completing on the
// mbarrier at `bar`'s offset in that CTA
__device__ __forceinline__ void bulk_g2s_multicast(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar,
                                                   uint16_t cta_mask) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;" ::"r"(
            smem_u32(smem_dst)),
        "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)), "h"(cta_mask)
        : "memory");
}
// 1-D bulk copy from this CTA's shared memory to another CTA's of the cluster (dst and bar: shared::cluster addresses,
// mapa), completing on that CTA's mbarrier
__device__ __forceinline__ void bulk_s2s_cluster(uint32_t dst, uint32_t src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "r"(src),
                 "r"(bytes), "r"(bar)
                 : "memory");
}
// generic-proxy writes (st.shared) -> visible to the async proxy (wgmma operand reads, bulk copies)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// named barrier over `count` threads (a multiple of 32); id 0 is __syncthreads
__device__ __forceinline__ void named_bar_sync(int id, int count) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// ---- programmatic dependent launch (PDL): the generator chain's kernels are launched with
// cudaLaunchAttributeProgrammaticStreamSerialization, so kernel N+1's CTAs may start -- barrier init and the weight
// stream of its first ring slots: everything that does not touch kernel N's output -- while kernel N's last wave is
// still running.  pdl_trigger(): "my dependents may be scheduled" (they still wait for this whole grid's completion and
// memory flush in pdl_wait()); pdl_wait(): executed by every thread that reads or writes activations, before it does.
// Both are no-ops in a launch without the attribute.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---- descriptors ------------------------------------------------------------------------------
// Shared-memory matrix descriptor of wgmma, no swizzle (layout type 0), K-major:
// [0,14) start >> 4 | [16,30) LBO >> 4 | [32,46) SBO >> 4 | [49,52) base offset = 0 | [62,64) layout = 0.
// descriptor = constant high part (LBO, SBO) | 14-bit start-address field
__device__ __forceinline__ uint64_t desc_template(uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) | ((uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32);
}
__device__ __forceinline__ uint64_t desc_at(uint64_t tmpl, uint32_t saddr) { return tmpl | (uint64_t)((saddr >> 4) & 0x3FFF); }

// ---- warpgroup MMA ------------------------------------------------------------------------------
// Every thread of the warpgroup executes these, converged.  Order per accumulator tile:
//   wgmma_fence() (registers written by ordinary instructions become visible to the MMA), wgmma_bf16() x n,
//   wgmma_commit(), wgmma_wait<k>() (at most k committed groups still in flight), then acc_fence() before the
//   registers are read or written by ordinary code.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMA window
template <int R>
__device__ __forceinline__ void acc_fence(float *d) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// thread `t` (0..127 of its warpgroup): row of accumulator element d[4k + 2h + e], and column of d[j]
__device__ __forceinline__ int frag_row(int t, int h) { return 16 * (t >> 5) + ((t & 31) >> 2) + 8 * h; }
__host__ __device__ constexpr int frag_col(int lane_q, int j) { return 8 * (j >> 2) + 2 * lane_q + (j & 1); }

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, both operands in shared memory (K-major descriptors), D in the N/2 registers
// d[0 .. N/2); scale_d = 0 overwrites D.  N = 32 on the first 16 registers of an N = 64 tile accumulates onto its first
// 32 columns (the register layout of a column block does not depend on N).
template <int N>
__device__ __forceinline__ void wgmma_bf16(float *d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d);
#define MG_D8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
template <> __device__ __forceinline__ void wgmma_bf16<32>(float *d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
                 : MG_D8(0), MG_D8(8)
                 : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_bf16<64>(float *d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
                 : MG_D8(0), MG_D8(8), MG_D8(16), MG_D8(24)
                 : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_bf16<128>(float *d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
                 : MG_D8(0), MG_D8(8), MG_D8(16), MG_D8(24), MG_D8(32), MG_D8(40), MG_D8(48), MG_D8(56)
                 : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_bf16<160>(float *d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %82, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n160k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79}, %80, %81, p, 1, 1, 0, 0;\n\t}"
                 : MG_D8(0), MG_D8(8), MG_D8(16), MG_D8(24), MG_D8(32), MG_D8(40), MG_D8(48), MG_D8(56), MG_D8(64), MG_D8(72)
                 : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_bf16<256>(float *d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, %128, %129, p, 1, 1, 0, 0;\n\t}"
                 : MG_D8(0), MG_D8(8), MG_D8(16), MG_D8(24), MG_D8(32), MG_D8(40), MG_D8(48), MG_D8(56), MG_D8(64), MG_D8(72), MG_D8(80), MG_D8(88), MG_D8(96), MG_D8(104), MG_D8(112), MG_D8(120)
                 : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
// The same instruction with its accumulator in two register arrays: columns [0, N/2) in d0[0 .. N/4), columns [N/2, N) in
// d1[0 .. N/4).  With B = [wh | wl] stacked along N (mg_layout.h, tc_stacked) one MMA leaves x * wh^T in d0 and x * wl^T
// in d1; scale_d applies to both.
template <int N>
__device__ __forceinline__ void wgmma_bf16_pair(float *d0, float *d1, uint64_t adesc, uint64_t bdesc, uint32_t scale_d);
#define MG_E8(i) "+f"(d1[i]), "+f"(d1[i + 1]), "+f"(d1[i + 2]), "+f"(d1[i + 3]), "+f"(d1[i + 4]), "+f"(d1[i + 5]), "+f"(d1[i + 6]), "+f"(d1[i + 7])
template <> __device__ __forceinline__ void wgmma_bf16_pair<64>(float *d0, float *d1, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    float *d = d0;
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
                 : MG_D8(0), MG_D8(8), MG_E8(0), MG_E8(8)
                 : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_bf16_pair<128>(float *d0, float *d1, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    float *d = d0;
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
                 : MG_D8(0), MG_D8(8), MG_D8(16), MG_D8(24), MG_E8(0), MG_E8(8), MG_E8(16), MG_E8(24)
                 : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
#undef MG_E8
#undef MG_D8

// ---- bf16 hi/lo split ----------------------------------------------------------------------------
// x ~= hi + lo with hi = bf16(x) (round-to-nearest), lo = bf16(x - hi): 16 significant bits, so the
// three-pass product xh*wh + xl*wh + xh*wl carries ~2^-16 relative error per term (SURVEY 0.4 measured
// 5e-6..1.5e-5 end to end, 100x inside the 1e-3 tolerance; single-pass bf16 or tf32 is not).
__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16 &hi, __nv_bfloat16 &lo) {
    hi = __float2bfloat16_rn(x);
    lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}
// packs two floats' hi parts / lo parts into two 32-bit words (element 0 in the low half)
__device__ __forceinline__ void split2_bf16(float x0, float x1, uint32_t &hi, uint32_t &lo) {
    __nv_bfloat162 h = __floats2bfloat162_rn(x0, x1);
    float2 hf = __bfloat1622float2(h);
    __nv_bfloat162 l = __floats2bfloat162_rn(x0 - hf.x, x1 - hf.y);
    hi = *reinterpret_cast<uint32_t *>(&h);
    lo = *reinterpret_cast<uint32_t *>(&l);
}

// ---- single-pass bf16 variant of a kernel configuration (mg_gen_forward_precision, MG_GEN_PRECISION_BF16) ----------
// The same tiles, shared-memory layout and packed blob as Cfg, but one pass (xh, wh) per product with fp32 accumulation:
// the converters store only the hi operand, and only the hi half of each weight chunk / slot is brought in (the lo half
// of the blob and the Xl / lo regions of shared memory are left unused; a stacked chunk, mg_layout.h tc_stacked, comes in
// whole and its lo rows are skipped by the descriptor).  A distinct type, so the instantiations have
// kernel symbols of their own ("resblock_tc_kernel<mg::tc::Bf16<mg::RbCfg<...>>>") in a profiler trace.
template <class Cfg>
struct Bf16 : Cfg {
    static constexpr bool ONEPASS = true;
};

}  // namespace tc
}  // namespace mg
