// PTX wrappers and epilogue helpers shared by the wgmma kernels (igemm_umma.cu, conv_tma.cu, dcn_tma.cu).  sm_90a.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace cp {
namespace umma {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// bounded wait: a protocol bug traps (reported as a CUDA launch failure) instead of hanging the device.  The slow path
// is call-free (a printf here costs a real ABI call: ~20 extra instructions and the spill code of every live register at
// each of the ~10 wait sites of a hot loop); build with -DCP_MBAR_DEBUG to get the diagnostic message back.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) {
#ifdef CP_MBAR_DEBUG
      printf("wgmma kernel: mbarrier watchdog (block %d thread %d bar %u parity %u)\n", blockIdx.x, threadIdx.x, bar, parity);
#endif
      __trap();
    }
  }
}
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
// named barrier of the 128 threads of one warpgroup (ids 1 .. 15; 0 is __syncthreads)
__device__ __forceinline__ void wg_bar_sync(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

// ---- wgmma: a warpgroup (128 threads) multiplies a 64-row A tile by an N-row B tile, both K-major in shared memory,
// into a register accumulator.  Fragment of thread t (warp w = t / 32, lane l): d[4 j + 2 i + c] holds row
// 16 w + l / 4 + 8 i, column 8 j + 2 (l % 4) + c.
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_tf32(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d);
template <int N>
__device__ __forceinline__ void wgmma_bf16(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d);
template <> __device__ __forceinline__ void wgmma_tf32<16>(float (&d)[8], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_tf32<32>(float (&d)[16], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_tf32<64>(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_tf32<128>(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_tf32<256>(float (&d)[128], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, %128, %129, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_bf16<16>(float (&d)[8], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_bf16<32>(float (&d)[16], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_bf16<64>(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_bf16<128>(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_bf16<256>(float (&d)[128], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, %128, %129, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(da), "l"(db), "r"(scale_d));
}

// Register-A form (tf32 only): thread t of warp w holds the A fragment of rows 16 w + l / 4 (+ 8), columns l % 4
// (+ 4) of the 64 x 8 slice (PTX ISA, wgmma .m64nNk8 A fragment): a[0] = (r, c), a[1] = (r + 8, c), a[2] = (r, c + 4),
// a[3] = (r + 8, c + 4).  The registers must stay untouched until the wgmma has been waited for.
template <int N>
__device__ __forceinline__ void wgmma_tf32_rs(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d);
template <> __device__ __forceinline__ void wgmma_tf32_rs<16>(float (&d)[8], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7}, {%8,%9,%10,%11}, %12, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_tf32_rs<32>(float (&d)[16], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, {%16,%17,%18,%19}, %20, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_tf32_rs<64>(float (&d)[32], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_tf32_rs<128>(float (&d)[64], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}

// One K block on the tensor cores: KS slices of 32 bytes (8 tf32 / 16 bf16 elements) of a 64-row A tile and a BN-row B
// tile.  X3: 3-term split a_lo b_hi + a_hi b_lo + a_hi b_hi (lo tiles at a_lo / b_lo descriptor units past the hi tiles),
// cross terms first.  fresh: the first product overwrites the accumulator.  Returns when the products are in `acc` and
// the operand tiles may be reused.
template <int BN, bool X3, bool BF16, int KS>
__device__ __forceinline__ void mma_kblock(float (&acc)[BN / 2], uint64_t da, uint64_t db, uint32_t a_lo, uint32_t b_lo,
                                           bool fresh) {
  wg_fence();
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) {
    const uint32_t sd = (fresh && ks == 0) ? 0u : 1u;
    if (X3) {
      wgmma_tf32<BN>(acc, da + a_lo + 2u * ks, db + 2u * ks, sd);
      wgmma_tf32<BN>(acc, da + 2u * ks, db + b_lo + 2u * ks, 1u);
    } else if (BF16) {
      wgmma_bf16<BN>(acc, da + 2u * ks, db + 2u * ks, sd);
    } else {
      wgmma_tf32<BN>(acc, da + 2u * ks, db + 2u * ks, sd);
    }
  }
  if (X3) {
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) wgmma_tf32<BN>(acc, da + 2u * ks, db + 2u * ks, 1u);
  }
  wg_commit();
  wg_wait<0>();
}

// Round to tf32 (10 mantissa bits), nearest, ties away from zero == cvt.rna.tf32.f32 for every finite input (the add
// carries into the exponent exactly like the rounding does; FLT_MAX rounds to inf either way).  ptxas expands the cvt
// into IADD + FSETP + SEL + LOP3 (NaN / inf preserved); activations are finite, so the two-instruction form is used:
// the hi / lo split of the 3-term product runs it 32 times per position and K block.
__device__ __forceinline__ float tf32_round(float x) {
  return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u);
}
// Four 8 x 8 b16 matrices; lanes 8 q .. 8 q + 7 give the row addresses of matrix q, register q of lane l gets bytes
// 4 (l % 4) .. + 4 of row l / 4 of matrix q: one tf32 element.
__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}

// One tf32x3 K block with A in registers: the 3-term split a_lo b_hi + a_hi b_lo + a_hi b_hi in mma_kblock's product
// order (cross terms first, slice by slice, then the hi products), so the results equal those of the shared-memory
// hi / lo A tiles.  A (this warpgroup's 64 rows, fp32) is read once per slice from shared memory into registers and
// split there; B keeps its hi tile at `db` and its lo tile `b_lo` descriptor units further.  The A tile is K-major with
// rows of 32 KS bytes (KS = 4: SWIZZLE_128B, KS = 2: SWIZZLE_64B), row 0 at `a_tile` (a multiple of the row size; the
// XOR comes from the address bits, as in make_desc).  wt: thread in the warpgroup.  fresh: the first product
// overwrites the accumulator.  Returns when the products are in `acc` and the operand tiles may be reused.
template <int BN, int KS>
__device__ __forceinline__ void mma_kblock_x3(float (&acc)[BN / 2], uint32_t a_tile, int wt, uint64_t db, uint32_t b_lo,
                                              bool fresh) {
  const uint32_t lane = (uint32_t)wt & 31u;
  // ldmatrix matrices 0..3 = (rows 0-7, k 0-3), (rows 8-15, k 0-3), (rows 0-7, k 4-7), (rows 8-15, k 4-7) of the warp's
  // 16 rows: the wgmma A fragment a[0..3]
  const uint32_t row = (uint32_t)(wt >> 5) * 16u + (lane & 7u) + ((lane >> 3) & 1u) * 8u;
  const uint32_t a_row = a_tile + row * (32u * KS);
  const uint32_t x = ((lane >> 4) << 4) ^ ((a_row >> 3) & (KS == 4 ? 0x70u : 0x30u));
  uint32_t hi[KS][4], lo[KS][4];
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) {
    ldsm_x4(hi[ks], a_row + (((uint32_t)ks << 5) ^ x));
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float v = __uint_as_float(hi[ks][j]);
      const float h = tf32_round(v);
      lo[ks][j] = __float_as_uint(tf32_round(v - h));
      hi[ks][j] = __float_as_uint(h);
    }
  }
  wg_fence();
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) {
    wgmma_tf32_rs<BN>(acc, lo[ks], db + 2u * ks, (fresh && ks == 0) ? 0u : 1u);
    wgmma_tf32_rs<BN>(acc, hi[ks], db + b_lo + 2u * ks, 1u);
  }
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) wgmma_tf32_rs<BN>(acc, hi[ks], db + 2u * ks, 1u);
  wg_commit();
  wg_wait<0>();
  // the tensor cores read the A registers until the wait: keep them live (and unchanged) up to here
#pragma unroll
  for (int ks = 0; ks < KS; ++ks)
#pragma unroll
    for (int j = 0; j < 4; ++j) asm volatile("" : "+r"(hi[ks][j]), "+r"(lo[ks][j]));
}

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));   // low half <- a
  return r;
}
__device__ __forceinline__ void st_shared_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ void st_shared_v4f(uint32_t addr, float a, float b, float c, float d) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ float4 ld_shared_v4f(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
  return v;
}

// ---- TMA tensor loads and shared-memory matrix descriptors (conv_tma.cu, dcn_tma.cu)
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, int c3, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];" ::"r"(dst),
      "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(bar)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int c0, int c1, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
               "l"(map), "r"(c0), "r"(c1), "r"(bar)
               : "memory");
}
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}

// wgmma shared-memory matrix descriptor, K-major and swizzled; `saddr` may be any multiple of 16 bytes.  The swizzle
// is a function of the shared-memory address bits [7,10) (like the one TMA applies when it writes the slab), so a matrix
// that starts at an arbitrary row of a slab needs no base-offset correction.
//   [0,14) start address >> 4, [16,30) leading byte offset >> 4 (unused when swizzled, 1), [32,46) stride byte offset >> 4
//   = distance of 8-row groups, [62,64) layout: 1 = SWIZZLE_128B, 2 = SWIZZLE_64B
// cslab = 32: 128-byte rows, SWIZZLE_128B, 8-row groups 1024 bytes apart;
// cslab = 16:  64-byte rows, SWIZZLE_64B,  8-row groups  512 bytes apart.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, int cslab) {
  const uint64_t sbo = cslab == 32 ? (1024 >> 4) : (512 >> 4);
  const uint64_t lay = cslab == 32 ? 1ull : 2ull;
  return (uint64_t)((saddr >> 4) & 0x3FFFu) | (1ull << 16) | (sbo << 32) | (lay << 62);
}

// ---------------------------------------------------------------------------------------------------------------
// The fused epilogue of NV consecutive columns of one output row: bias, residual (before or after the ReLU), ReLU,
// optional tf32 rounding, then an NHWC store (16-byte stores along the row) or an NCHW store.
struct EpiParams {
  const float* bias;
  const float* residual;
  int resStride, relu, res_after_relu, round_tf32;
  float* out;
  int outStride, out_nchw;
  int Cout, CoutPad, H, W;   // Cout/H/W: NCHW addressing; CoutPad: length of the bias vector
};

template <int NV>
__device__ __forceinline__ void epilogue_row(const EpiParams& e, float (&vv)[NV], bool valid, int m, int n, int oy, int ox,
                                             int col0, int col_end) {
#pragma unroll
  for (int j = 0; j < NV; ++j)
    if (col0 + j < e.CoutPad) vv[j] += __ldg(e.bias + col0 + j);
  if (e.residual && valid && !e.res_after_relu) {
    const float* r = e.residual + (size_t)m * e.resStride + col0;
#pragma unroll
    for (int j = 0; j < NV; ++j)
      if (col0 + j < col_end) vv[j] += __ldg(r + j);
  }
  if (e.relu) {
#pragma unroll
    for (int j = 0; j < NV; ++j) vv[j] = fmaxf(vv[j], 0.f);
  }
  if (e.residual && valid && e.res_after_relu) {
    const float* r = e.residual + (size_t)m * e.resStride + col0;
#pragma unroll
    for (int j = 0; j < NV; ++j)
      if (col0 + j < col_end) vv[j] += __ldg(r + j);
  }
  if (e.round_tf32) {
#pragma unroll
    for (int j = 0; j < NV; ++j) vv[j] = tf32_round(vv[j]);
  }
  if (!valid) return;
  if (e.out_nchw) {
#pragma unroll
    for (int j = 0; j < NV; ++j)
      if (col0 + j < col_end) e.out[(((size_t)n * e.Cout + col0 + j) * e.H + oy) * e.W + ox] = vv[j];
  } else {
    float* o = e.out + (size_t)m * e.outStride + col0;
#pragma unroll
    for (int j = 0; j < NV; j += 4) {
      if (col0 + j + 3 < col_end) {
        *reinterpret_cast<float4*>(o + j) = make_float4(vv[j], vv[j + 1], vv[j + 2], vv[j + 3]);
      } else {
#pragma unroll
        for (int t = 0; t < 4; ++t)
          if (col0 + j + t < col_end) o[j + t] = vv[j + t];
      }
    }
  }
}

// Split-K, second half (conv_tma_splitk_finish, dcn_tma_splitk_finish): one thread per (tile row i, 4 columns) of an
// (m, n) tile adds the ksplit partial sums ([mn tile][split][BN / 4][rows] float4, row-fastest: coalesced) in split
// order and runs the epilogue.  row_at(mn, i, &n, &oy, &ox) maps the row to its output position (false: none).  MULTI
// (several models in the launch): image n takes the bias of model n / p.ipm.
template <bool MULTI, class Params, class RowAt>
__device__ __forceinline__ void splitk_finish(const Params& p, int rows, long long mn_tiles, RowAt row_at) {
  griddep_launch_dependents();
  griddep_wait();
  const int G = p.BN >> 2;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= mn_tiles * G * rows) return;
  const int i = (int)(idx % rows);
  const int c4 = (int)((idx / rows) % G);
  const long long mn = idx / ((long long)rows * G);
  const float4* src = reinterpret_cast<const float4*>(p.part) + ((size_t)mn * p.ksplit * G + c4) * rows + i;
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int q = 0; q < p.ksplit; ++q) {
    const float4 v = __ldcg(src + (size_t)q * G * rows);
    a.x += v.x;
    a.y += v.y;
    a.z += v.z;
    a.w += v.w;
  }
  int n, oy, ox;
  if (!row_at(mn, i, &n, &oy, &ox)) return;
  const int n_tile = (int)(mn % (p.CoutPad / p.BN));
  const EpiParams e{MULTI ? p.bias + (size_t)(n / p.ipm) * p.wstride : p.bias, p.residual, p.resStride, p.relu, p.res_after_relu, p.round_tf32, p.out, p.outStride, p.out_nchw,
                    p.Cout, p.CoutPad, p.H, p.W};
  float v[4] = {a.x, a.y, a.z, a.w};
  epilogue_row<4>(e, v, true, (n * p.H + oy) * p.W + ox, n, oy, ox, n_tile * p.BN + c4 * 4, min(p.Cout, (n_tile + 1) * p.BN));
}

// Row-wise drain of a warpgroup's 64 x BN wgmma accumulator: 32 columns at a time go through `stage` (64 x 33 floats of
// shared memory owned by the warpgroup); thread t then holds row t / 2, columns 16 (t % 2) .. + 16 of the chunk and
// calls fn(row, first column, values).  fn runs for every thread and chunk, also where the columns lie past BN (BN = 16).
constexpr uint32_t DRAIN_STAGE_BYTES = 64u * 33u * 4u;
template <int BN, class Fn>
__device__ __forceinline__ void drain_rows(const float (&acc)[BN / 2], float* stage, int wt, int bar_id, Fn&& fn) {
  const int r0 = (wt >> 5) * 16 + ((wt & 31) >> 2), cq = (wt & 3) * 2;
#pragma unroll
  for (int c0 = 0; c0 < BN; c0 += 32) {
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      if (j * 8 >= c0 && j * 8 < c0 + 32) {
        const int c = j * 8 - c0 + cq;
        stage[r0 * 33 + c] = acc[4 * j];
        stage[r0 * 33 + c + 1] = acc[4 * j + 1];
        stage[(r0 + 8) * 33 + c] = acc[4 * j + 2];
        stage[(r0 + 8) * 33 + c + 1] = acc[4 * j + 3];
      }
    }
    wg_bar_sync(bar_id);
    const int r = wt >> 1, h = wt & 1;
    float v[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = (c0 + 16 * h + j < BN) ? stage[r * 33 + 16 * h + j] : 0.f;
    fn(r, c0 + 16 * h, v);
    wg_bar_sync(bar_id);
  }
}

// Largest wgmma N (16 .. 256, a power of two, <= cap) that divides CoutPad (16, 32 or a multiple of 64).
inline int wgmma_tile_n(int CoutPad, int cap) {
  for (int n = 256; n >= 16; n >>= 1)
    if (n <= cap && CoutPad % n == 0) return n;
  return 0;
}

}  // namespace umma
}  // namespace cp
