// Device helpers of the warp-autonomous element pipelines (b2p_hex_nd3.cu, b2p_hex_h1v3.cu):
// mbarrier + TMA bulk copies, cp.async staging, signed-restriction gather/scatter fast paths.
#pragma once
#include "b2p_contract.cuh"

namespace b2p
{

#ifdef B2P_EMU
// Host-thread SIMT emulation (tests/emu/cuda_emu.hpp, test infrastructure): same protocol, no PTX.
inline void mbar_init(uint64_t *bar, int count) { ::cuda_emu::mbar_init(bar, count); }
inline void mbar_expect_tx(uint64_t *bar, uint32_t bytes) { ::cuda_emu::mbar_expect_tx(bar, bytes); }
inline void tma_bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) { ::cuda_emu::tma_bulk_g2s(dst, src, bytes, bar); }
inline uint64_t l2_evict_first_policy() { return 0; }
inline void tma_bulk_g2s_hint(void *dst, const void *src, uint32_t bytes, uint64_t *bar, uint64_t)
{
  ::cuda_emu::tma_bulk_g2s(dst, src, bytes, bar);
}
inline void mbar_wait(uint64_t *bar, uint32_t parity) { ::cuda_emu::mbar_wait(bar, parity); }
inline void cp_async8(void *dst, const void *src) { ::cuda_emu::cp_async(dst, src, 8); }
inline void cp_async_commit() { ::cuda_emu::cp_async_commit(); }
template <int N>
inline void cp_async_wait()
{
  ::cuda_emu::cp_async_wait(N);
}
inline void fence_proxy_async() {}
inline unsigned long long ld_acquire_sys_u64(const unsigned long long *p)
{
  ::cuda_emu::yield();  // (spin loops on the halo flags: let the other fibers run)
  return *(const volatile unsigned long long *)p;
}
inline void st_release_sys_u64(unsigned long long *p, unsigned long long v)
{
  *(volatile unsigned long long *)p = v;
  ::cuda_emu::st().events++;
}
inline void dmma884(double &c0, double &c1, double a, double b) { ::cuda_emu::dmma884(c0, c1, a, b); }
inline void griddep_wait() {}               // launches are synchronous in the emulation
inline void griddep_launch_dependents() {}
inline void red_add_f64_if(double *addr, double v, bool pred)
{
  if (pred) atomicAdd(addr, v);
}
#else
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, int count)
{
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar)
{
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// L2 policy for data an element kernel reads exactly once per launch (q-data, restriction indices, coefficient blocks):
// their lines are evicted first, so the stream does not push out the lines that are used again -- x and y, which every
// element around a dof gathers and scatter-adds, and whatever the caller keeps in L2 between launches.
__device__ __forceinline__ uint64_t l2_evict_first_policy()
{
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ void tma_bulk_g2s_hint(void *dst, const void *src, uint32_t bytes, uint64_t *bar, uint64_t policy)
{
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
  uint32_t ok = 0;
  while (!ok)
  {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  }
}

__device__ __forceinline__ void cp_async8(void *dst, const void *src)
{
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait()
{
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ unsigned long long ld_acquire_sys_u64(const unsigned long long *p)
{
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys_u64(unsigned long long *p, unsigned long long v)
{
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// Programmatic dependent launch (PDL): a kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may start
// while its predecessor in the stream still runs; griddepcontrol.wait blocks until the predecessor has completed and its
// writes are visible (returns at once when the kernel was launched normally); the predecessor releases its dependent
// early with griddepcontrol.launch_dependents.
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void griddep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
// FP64 tensor-core MMA, D(8x8) = A(8x4) B(4x8) + C: a = A[lane/4][lane%4], b = B[lane%4][lane/4],
// {c0, c1} = C[lane/4][2 (lane%4) + {0, 1}]  (SASS DMMA.8x8x4)
__device__ __forceinline__ void dmma884(double &c0, double &c1, double a, double b)
{
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
#endif

// Staged dof value with the restriction's sign (masked / padded slots were staged as zero):
// the sign bit of the index is XORed into the high word of the value.
__device__ __forceinline__ double staged(const int32_t *cI, const double *cU, int pos, bool valid)
{
  const int32_t gi = cI[pos];
  const double v = cU[pos];
  int hi = __double2hiint(v) ^ (gi & (int)0x80000000);
  const double r = __hiloint2double(hi, __double2loint(v));
  return valid ? r : 0.0;
}
// Same with the index row and the staged values at different positions (several vector parts of one element
// share the element's index row).
__device__ __forceinline__ double staged2(const int32_t *cI, int ipos, const double *cU, int upos, bool valid)
{
  const int32_t gi = cI[ipos];
  const double v = cU[upos];
  int hi = __double2hiint(v) ^ (gi & (int)0x80000000);
  const double r = __hiloint2double(hi, __double2loint(v));
  return valid ? r : 0.0;
}
// |index| of a signed restriction entry (-1 - gi == ~gi for negative entries)
__device__ __forceinline__ int32_t abs_idx(int32_t gi) { return gi ^ (gi >> 31); }
// Predicated RED.F64 of value (with the entry's sign) at y[|gi|]; masked entries are skipped.
__device__ __forceinline__ void scatter_fast(double *y, int32_t gi, double v)
{
  const int hi = __double2hiint(v) ^ (gi & (int)0x80000000);
  const double sv = __hiloint2double(hi, __double2loint(v));
  double *addr = y + (uint32_t)abs_idx(gi);
#ifdef B2P_EMU
  red_add_f64_if(addr, sv, gi != (int32_t)0x80000000);
#else
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.s32 p, %2, 0x80000000;\n"
      "@p red.global.add.f64 [%0], %1;\n"
      "}\n" ::"l"(addr),
      "d"(sv), "r"(gi)
      : "memory");
#endif
}


// Same with the L-vector in two pieces (owned part in y, ghosts in sp.yg): one compare + select on
// 32-bit indices picks the base, the rest is the fast path.
__device__ __forceinline__ void scatter_fast_split(double *y, const VSplit &sp, int32_t gi, double v)
{
  const int hi = __double2hiint(v) ^ (gi & (int)0x80000000);
  const double sv = __hiloint2double(hi, __double2loint(v));
  const uint32_t a = (uint32_t)abs_idx(gi), no = (uint32_t)sp.n_owned;
  double *addr = (a < no) ? y + a : sp.yg + (a - no);
#ifdef B2P_EMU
  red_add_f64_if(addr, sv, gi != (int32_t)0x80000000);
#else
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.s32 p, %2, 0x80000000;\n"
      "@p red.global.add.f64 [%0], %1;\n"
      "}\n" ::"l"(addr),
      "d"(sv), "r"(gi)
      : "memory");
#endif
}
__device__ __forceinline__ const double *split_src_fast(const double *x, const VSplit &sp, int32_t a)
{
  const uint32_t ua = (uint32_t)a, no = (uint32_t)sp.n_owned;
  return (ua < no) ? x + ua : sp.xg + (ua - no);
}

}  // namespace b2p
