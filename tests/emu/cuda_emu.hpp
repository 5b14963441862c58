// TEST INFRASTRUCTURE ONLY -- never part of libb2p.so.
//
// SIMT-on-fibers emulation used to execute the UNMODIFIED kernel sources of palace_b200/csrc on the CPU
// (B2P_EMU_TESTS=1 python -m pytest tests -m gpu, see tests/emu/emu_mode.py): every CUDA thread of a block is a
// user-level fiber with its own stack; __syncthreads / __syncwarp are real barriers between fibers (a fiber that
// has exited no longer counts, as on the device); shuffles and mma.sync exchange values through per-warp
// mailboxes using the PTX fragment layouts; TMA bulk copies and mbarriers follow their phase/parity protocol;
// cp.async copies are deferred until the matching wait, so a missing wait reads stale data; shared memory and
// "device" allocations are poisoned. Fibers of a barrier interval run one after the other (order selectable with
// B2P_EMU_ORDER=fwd|rev|rand), so a missing barrier between a producer and a consumer phase shows up as stale
// data for some lane order. Blocks run one at a time. This validates indexing, data flow, synchronisation protocol
// and arithmetic of a kernel before it is run on an H100; it says nothing about performance. The product never
// links or loads it: B2P_EMU is defined only by tests/emu/Makefile.
#pragma once
#include <sys/mman.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <random>
#include <vector>

#if !defined(__x86_64__)
#error "tests/emu: the fiber switch is written for x86-64"
#endif

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline __attribute__((always_inline))
#define __launch_bounds__(...)
#define __grid_constant__
#define __restrict__ __restrict
#define __align__(n) alignas(n)
#define __shared__ static /* blocks run one at a time: one instance per kernel instantiation is one per block */

struct uint3
{
  unsigned x, y, z;
};
struct dim3
{
  unsigned x, y, z;
  dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct alignas(16) double2
{
  double x, y;
};
inline double2 make_double2(double x, double y) { return double2{x, y}; }

extern "C" void b2p_emu_switch(void **save_sp, void *new_sp);
#ifdef B2P_EMU_DEFINE_SWITCH
asm(R"(
.text
.globl b2p_emu_switch
.type b2p_emu_switch,@function
b2p_emu_switch:
  pushq %rbp
  pushq %rbx
  pushq %r12
  pushq %r13
  pushq %r14
  pushq %r15
  movq %rsp, (%rdi)
  movq %rsi, %rsp
  popq %r15
  popq %r14
  popq %r13
  popq %r12
  popq %rbx
  popq %rbp
  ret
.size b2p_emu_switch,.-b2p_emu_switch
)");
#endif

namespace cuda_emu
{
struct Bar
{
  int expected = 0, arrived = 0;
  unsigned gen = 0;
};
struct Warp
{
  Bar bar;
  alignas(16) unsigned char mail[32][16];
  std::vector<std::pair<unsigned, Bar>> sub;  // barriers of partial member masks (__shfl_sync with a subset of the lanes)
  Bar &bar_for(unsigned mask)
  {
    if (mask == 0xffffffffu) return bar;
    for (auto &m : sub)
      if (m.first == mask) return m.second;
    Bar b;
    b.expected = __builtin_popcount(mask);
    sub.emplace_back(mask, b);
    return sub.back().second;
  }
};
struct Copy
{
  void *dst;
  const void *src;
  size_t n;
};
struct Fiber
{
  void *sp = nullptr;
  unsigned char *stack = nullptr;
  bool done = false;
  int lane = 0;
  Warp *warp = nullptr;
  uint3 tidx{0, 0, 0};
  std::vector<std::vector<Copy>> groups;  // cp.async groups in flight
  std::vector<Copy> open;
};
struct Block
{
  Bar bar;
  std::vector<Warp> warps;
  std::vector<unsigned char> smem;
  std::vector<Fiber> fibers;
  const std::function<void()> *body = nullptr;
};
struct State
{
  Fiber *cur = nullptr;
  Block *blk = nullptr;
  void *sched_sp = nullptr;
  uint3 bidx{0, 0, 0};
  dim3 bdim, gdim;
  unsigned long events = 0;  // progress counter for the deadlock watchdog
  std::vector<unsigned char *> free_stacks;
};
State &st();
constexpr size_t STACK_BYTES = 512 * 1024;

inline void yield() { b2p_emu_switch(&st().cur->sp, st().sched_sp); }
inline void *dyn_smem() { return st().blk->smem.data(); }

inline void bar_wait(Bar &b)
{
  const unsigned g = b.gen;
  if (++b.arrived >= b.expected)
  {
    b.arrived = 0;
    b.gen++;
    st().events++;
    return;
  }
  while (b.gen == g) yield();
}
inline void bar_drop(Bar &b)
{
  b.expected--;
  if (b.expected > 0 && b.arrived >= b.expected)
  {
    b.arrived = 0;
    b.gen++;
    st().events++;
  }
}
void fiber_entry();
void launch(dim3 grid, dim3 block, size_t shmem, const std::function<void()> &body);

#ifdef B2P_EMU_DEFINE_SWITCH
State &st()
{
  static thread_local State s;
  return s;
}
void fiber_entry()
{
  State &s = st();
  (*s.blk->body)();
  Fiber *f = st().cur;
  f->done = true;
  st().events++;
  // an exited thread no longer takes part in barriers (as on the device)
  bar_drop(f->warp->bar);
  bar_drop(st().blk->bar);
  b2p_emu_switch(&f->sp, st().sched_sp);
  std::abort();  // never resumed
}
static unsigned char *get_stack(State &s)
{
  if (!s.free_stacks.empty())
  {
    unsigned char *p = s.free_stacks.back();
    s.free_stacks.pop_back();
    return p;
  }
  void *p = mmap(nullptr, STACK_BYTES, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
  if (p == MAP_FAILED)
  {
    std::perror("cuda_emu: mmap fiber stack");
    std::abort();
  }
  return (unsigned char *)p;
}
static void start_fiber(State &s, Fiber &f)
{
  f.stack = get_stack(s);
  uintptr_t top = ((uintptr_t)f.stack + STACK_BYTES) & ~(uintptr_t)15;
  void **sp = (void **)(top - 64);  // [r15 r14 r13 r12 rbx rbp | return address | pad]
  for (int i = 0; i < 6; i++) sp[i] = nullptr;
  sp[6] = (void *)&fiber_entry;
  sp[7] = nullptr;
  f.sp = sp;
}
void launch(dim3 grid, dim3 block, size_t shmem, const std::function<void()> &body)
{
  State &s = st();
  if (s.cur)
  {
    std::fprintf(stderr, "cuda_emu: nested kernel launch\n");
    std::abort();
  }
  const int nt = (int)(block.x * block.y * block.z), nw = (nt + 31) / 32;
  static const char *order_env = std::getenv("B2P_EMU_ORDER");
  const int order = !order_env ? 0 : (order_env[0] == 'r' && order_env[1] == 'e') ? 1 : (order_env[0] == 'r') ? 2 : 0;
  static thread_local std::mt19937 rng(12345);
  s.bdim = block;
  s.gdim = grid;
  for (unsigned bz = 0; bz < grid.z; bz++)
    for (unsigned by = 0; by < grid.y; by++)
      for (unsigned bx = 0; bx < grid.x; bx++)
      {
        Block blk;
        blk.body = &body;
        blk.smem.assign(shmem + 64, 0xCD);  // poison: uninitialised shared memory is not zero on the device either
        blk.bar.expected = nt;
        blk.warps.resize(nw);
        for (int w = 0; w < nw; w++) blk.warps[w].bar.expected = std::min(32, nt - 32 * w);
        blk.fibers.resize(nt);
        s.blk = &blk;
        s.bidx = uint3{bx, by, bz};
        std::vector<int> live(nt);
        for (int t = 0; t < nt; t++)
        {
          Fiber &f = blk.fibers[t];
          f.lane = t % 32;
          f.warp = &blk.warps[t / 32];
          f.tidx = uint3{(unsigned)t % block.x, ((unsigned)t / block.x) % block.y, (unsigned)t / (block.x * block.y)};
          live[t] = t;
        }
        unsigned long last_events = s.events;
        long idle_sweeps = 0;
        while (!live.empty())
        {
          if (order == 1)
            std::sort(live.begin(), live.end(), std::greater<int>());
          else if (order == 2)
            std::shuffle(live.begin(), live.end(), rng);
          for (int t : live)
          {
            Fiber &f = blk.fibers[t];
            if (!f.sp) start_fiber(s, f);
            s.cur = &f;
            b2p_emu_switch(&s.sched_sp, f.sp);
            s.cur = nullptr;
            if (f.done)
            {
              s.free_stacks.push_back(f.stack);
              f.stack = nullptr;
            }
          }
          live.erase(std::remove_if(live.begin(), live.end(), [&](int t) { return blk.fibers[t].done; }), live.end());
          if (order == 0) std::sort(live.begin(), live.end());
          if (s.events == last_events)
          {
            if (++idle_sweeps > 2000000)
            {
              std::fprintf(stderr, "cuda_emu: no progress in block (%u,%u,%u): %zu threads stuck (deadlocked barrier / mbarrier / flag wait)\n", bx,
                           by, bz, live.size());
              std::abort();
            }
          }
          else
          {
            idle_sweeps = 0;
            last_events = s.events;
          }
        }
        s.blk = nullptr;
      }
}
#endif

template <typename T>
inline T exchange(T v, int src_lane, unsigned mask = 0xffffffffu)
{
  static_assert(sizeof(T) <= 16, "");
  Fiber *f = st().cur;
  Warp *w = f->warp;
  if (!((mask >> f->lane) & 1u) || !((mask >> (src_lane & 31)) & 1u))
  {
    std::fprintf(stderr, "cuda_emu: shuffle with member mask %08x by lane %d from lane %d: both must be named in the mask\n", mask, f->lane,
                 src_lane & 31);
    std::abort();
  }
  std::memcpy(w->mail[f->lane], &v, sizeof(T));
  bar_wait(w->bar_for(mask));
  T r;
  std::memcpy(&r, w->mail[src_lane & 31], sizeof(T));
  bar_wait(w->bar_for(mask));
  return r;
}
// mma.sync.m8n8k4 f64: A[8x4] row-major fragment a = A[lane/4][lane%4], B[4x8] b = B[lane%4][lane/4],
// C/D[8x8] {c0, c1} = C[lane/4][2*(lane%4) + {0,1}]   (PTX ISA, "Matrix fragments for mma.m8n8k4 with .f64")
inline void dmma884(double &c0, double &c1, double a, double b)
{
  Fiber *f = st().cur;
  Warp *w = f->warp;
  const int lane = f->lane;
  double ab[2] = {a, b};
  std::memcpy(w->mail[lane], ab, 16);
  bar_wait(w->bar);
  const int g = lane / 4, t = lane % 4;
  for (int r = 0; r < 2; r++)
  {
    const int col = 2 * t + r;
    double s = r ? c1 : c0;
    for (int k = 0; k < 4; k++)
    {
      double A, B;
      std::memcpy(&A, w->mail[4 * g + k], 8);        // A[g][k] lives in lane 4g + k
      std::memcpy(&B, w->mail[4 * col + k] + 8, 8);  // B[k][col] lives in lane 4col + k
      s = std::fma(A, B, s);
    }
    (r ? c1 : c0) = s;
  }
  bar_wait(w->bar);
}

// mbarrier model (arrival count 1 + transaction bytes): the 64-bit word holds {completed phases : 32, pending tx : 32}
inline void mbar_init(uint64_t *bar, int) { *bar = 0; }
inline void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
  *bar += bytes;
  if (bytes == 0)
  {
    *bar += 1ull << 32;
    st().events++;
  }
}
inline void tma_bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar)
{
  if ((reinterpret_cast<uintptr_t>(dst) & 15) || (reinterpret_cast<uintptr_t>(src) & 15) || (bytes & 15))
  {
    std::fprintf(stderr, "cuda_emu: cp.async.bulk needs 16-byte aligned src / dst / size (dst %p src %p bytes %u)\n", dst, src, bytes);
    std::abort();
  }
  std::memcpy(dst, src, bytes);
  if ((uint32_t)*bar < bytes)
  {
    std::fprintf(stderr, "cuda_emu: complete_tx of %u bytes exceeds the expected transaction count %u\n", bytes, (uint32_t)*bar);
    std::abort();
  }
  *bar -= bytes;
  if ((uint32_t)*bar == 0)
  {
    *bar += 1ull << 32;  // phase complete
    st().events++;
  }
}
inline void mbar_wait(uint64_t *bar, uint32_t parity)
{
  // wait(parity) returns once the phase with that parity has completed
  while (((*bar >> 32) & 1u) == parity) yield();
}
inline void cp_async(void *dst, const void *src, size_t n) { st().cur->open.push_back({dst, src, n}); }
inline void cp_async_commit()
{
  Fiber *f = st().cur;
  f->groups.push_back(std::move(f->open));
  f->open.clear();
}
inline void cp_async_wait(int keep)
{
  Fiber *f = st().cur;
  while ((int)f->groups.size() > keep)
  {
    for (auto &c : f->groups.front()) std::memcpy(c.dst, c.src, c.n);
    f->groups.erase(f->groups.begin());
  }
}
}  // namespace cuda_emu

#define threadIdx (::cuda_emu::st().cur->tidx)
#define blockIdx (::cuda_emu::st().bidx)
#define blockDim (::cuda_emu::st().bdim)
#define gridDim (::cuda_emu::st().gdim)

inline void __syncthreads() { ::cuda_emu::bar_wait(::cuda_emu::st().blk->bar); }
inline void __syncwarp(unsigned = 0xffffffffu) { ::cuda_emu::bar_wait(::cuda_emu::st().cur->warp->bar); }
template <typename T>
inline T __shfl_xor_sync(unsigned mask, T v, int m)
{
  return ::cuda_emu::exchange(v, ::cuda_emu::st().cur->lane ^ m, mask);
}
template <typename T>
inline T __shfl_xor(T v, int m)
{
  return ::cuda_emu::exchange(v, ::cuda_emu::st().cur->lane ^ m);
}
template <typename T>
inline T __shfl_sync(unsigned mask, T v, int src)
{
  return ::cuda_emu::exchange(v, src, mask);
}
template <typename T>
inline T __ldg(const T *p)
{
  return *p;
}
template <typename T>
inline T __ldcv(const T *p)
{
  return *(const volatile T *)p;
}
inline void __threadfence_system() {}
inline void __threadfence() {}
inline int __double2hiint(double v)
{
  uint64_t u;
  std::memcpy(&u, &v, 8);
  return (int)(u >> 32);
}
inline int __double2loint(double v)
{
  uint64_t u;
  std::memcpy(&u, &v, 8);
  return (int)(u & 0xffffffffu);
}
inline double __hiloint2double(int hi, int lo)
{
  uint64_t u = ((uint64_t)(uint32_t)hi << 32) | (uint32_t)lo;
  double v;
  std::memcpy(&v, &u, 8);
  return v;
}
template <typename T>
inline T atomicAdd(T *p, T v)
{
  T old = *p;
  *p = old + v;
  return old;
}
using std::max;
using std::min;
inline double rsqrt(double x) { return 1.0 / std::sqrt(x); }
