// Baseline JPEG decode on the device (cp_jpeg_parse / cp_jpeg_decode), bit for bit cv2.imdecode: one launch per phase
// for a batch of frames of mixed sizes.  The arithmetic of every phase is jpeg_core.h, shared with the host restatement
// the tests pin against cv2.
//
//   1. jpeg_prep       scan preparation, one CTA per frame: drops stuffed 0x00 and fill bytes by a prefix sum over the
//                      uploaded bytes, cuts the scan at RSTn into restart segments and checks their numbering; then
//                      places each segment's subsequences (jpeg_subs fills the slot table).
//   2. jpeg_sync       self-synchronising Huffman decode (Weissenberger & Schmidt, ICPP 2018; the JPEG form, HiPC 2021):
//                      one thread per subsequence of subseq_words 32-bit words decodes from a guessed state (bit
//                      position, block in the MCU, zig-zag index) to the first symbol boundary in the next subsequence.
//                      A CTA re-decodes from its predecessors' exits until none changes; a round ends with each CTA
//                      handing its last exit to the next CTA.  The host repeats rounds until no handed-on state
//                      changes; subsequence 0 of a segment starts exact, so every round fixes at least one more CTA.
//   3. jpeg_scan       exclusive prefix sum of the blocks each subsequence begins.
//   4. jpeg_emit       the final pass: int16 coefficients in natural order and the DC differences; the only phase
//                      that reports a bitstream error.
//   5. jpeg_dc         DC prediction, a prefix sum per component segmented at each restart.
//   6. jpeg_idct       dequantisation and the islow IDCT into per-component uint8 planes.
//   7. jpeg_color      up-sampling, YCbCr -> BGR and the EXIF orientation, uint8 BGR at the caller's offset.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <string>
#include <vector>

#include "common.cuh"
#include "jpeg_core.h"

namespace cp {
namespace jpeg {
namespace {

constexpr int kDefaultSubseqWords = 8;
constexpr int kPrepThreads = 1024;
constexpr int kSyncThreads = 128;

struct Job {
  int64_t raw, nraw;       // the scan's bytes in d_bytes
  int64_t comp;            // its compacted bytes in the workspace
  int64_t sub0, nsub;      // subsequence slots
  int64_t blk0;            // first block of the coefficient buffer
  int64_t plane[3];        // component planes
  int64_t out;             // BGR output offset
  int32_t seg0, nseg;      // restart segments
};

struct Seg {
  uint32_t begin, end;     // compacted bytes, relative to the frame's
  int64_t first_sub;       // global slot of subsequence 0
  int32_t nsub, frame, index;
};

struct Layout {
  std::vector<Job> jobs;
  int64_t nseg = 0, nsub = 0, nblocks = 0, ncomp = 0, nplane = 0;
  int64_t maxblocks = 0, maxpix = 0;
  size_t off_hdr, off_job, off_seg, off_subseg, off_state, off_bnd, off_cnt, off_scan, off_flag, off_comp, off_diff,
      off_coef, off_plane, total;
};

size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

Layout layout(const cp_jpeg_header* hs, int B, int words) {
  Layout L;
  L.jobs.resize(B);
  for (int b = 0; b < B; ++b) {
    const cp_jpeg_header& h = hs[b];
    const SlotCap need = frame_need(h, words);
    Job& j = L.jobs[b];
    j.nraw = h.scan_end - h.scan_begin;
    j.comp = L.ncomp;
    L.ncomp += need.comp;
    j.seg0 = (int32_t)L.nseg;
    j.nseg = (int32_t)need.nseg;
    L.nseg += j.nseg;
    j.sub0 = L.nsub;
    j.nsub = need.nsub;
    L.nsub += j.nsub;
    j.blk0 = L.nblocks;
    int64_t nb = need.nblocks;
    L.nblocks += nb;
    if (nb > L.maxblocks) L.maxblocks = nb;
    for (int c = 0; c < 3; ++c) {
      j.plane[c] = L.nplane;
      if (c < h.ncomp) L.nplane += (int64_t)plane_w(h, c) * plane_h(h, c);
    }
    int64_t pix = (int64_t)h.out_h * h.out_w;
    if (pix > L.maxpix) L.maxpix = pix;
  }
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o += align256(bytes); return r; };
  L.off_hdr = take(sizeof(cp_jpeg_header) * B);
  L.off_job = take(sizeof(Job) * B);
  L.off_seg = take(sizeof(Seg) * L.nseg);
  L.off_subseg = take(sizeof(int32_t) * L.nsub);
  L.off_state = take(sizeof(uint64_t) * L.nsub);
  L.off_bnd = take(sizeof(uint64_t) * L.nsub * 2);
  L.off_cnt = take(sizeof(int32_t) * L.nsub);
  L.off_scan = take(sizeof(int32_t) * L.nsub);
  L.off_flag = take(sizeof(int32_t) * 4);
  L.off_comp = take(L.ncomp);
  L.off_diff = take(sizeof(int32_t) * L.nblocks);
  L.off_coef = take(sizeof(int16_t) * 64 * L.nblocks);
  L.off_plane = take(L.nplane);
  L.total = o;
  return L;
}

// The workspace of cp_jpeg_decode_slots_dev: slot s owns fixed regions of its capacity (slot_capacity of its decoded
// size, max_bytes and the subsequence length), so every grid and offset is known when a graph is built.  base[s] holds
// the slot's regions as a Job (raw: its encoded bytes in d_bytes, at the prefix sum of max_bytes; plane[0]: its planes).
struct SlotLayout {
  std::vector<Job> base;
  int64_t nseg = 0, nsub = 0, nblocks = 0, nplane = 0, ncomp = 0, raw = 0, maxblocks = 0, maxpix = 0, nctas = 0;
  size_t off_seg, off_subseg, off_state, off_cnt, off_scan, off_ticket, off_pub, off_comp, off_diff, off_coef,
      off_plane, total;
};

SlotLayout slot_layout(int S, const int32_t* hw, const int64_t* max_bytes, int words) {
  SlotLayout L;
  L.base.resize(S);
  for (int s = 0; s < S; ++s) {
    SlotCap c = slot_capacity(hw[2 * s], hw[2 * s + 1], max_bytes[s], words);
    Job& j = L.base[s];
    memset(&j, 0, sizeof(j));
    j.raw = L.raw;
    L.raw += max_bytes[s];
    j.comp = L.ncomp;
    L.ncomp += c.comp;
    j.seg0 = (int32_t)L.nseg;
    L.nseg += c.nseg;
    j.sub0 = L.nsub;
    L.nsub += c.nsub;
    j.blk0 = L.nblocks;
    L.nblocks += c.nblocks;
    j.plane[0] = L.nplane;
    L.nplane += c.nplane;
    if (c.nblocks > L.maxblocks) L.maxblocks = c.nblocks;
    int64_t pix = (int64_t)hw[2 * s] * hw[2 * s + 1];
    if (pix > L.maxpix) L.maxpix = pix;
  }
  L.nctas = (L.nsub + kSyncThreads - 1) / kSyncThreads;
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o += align256(bytes); return r; };
  L.off_seg = take(sizeof(Seg) * L.nseg);
  L.off_subseg = take(sizeof(int32_t) * L.nsub);
  L.off_state = take(sizeof(uint64_t) * L.nsub);
  L.off_cnt = take(sizeof(int32_t) * L.nsub);
  L.off_scan = take(sizeof(int32_t) * L.nsub);
  L.off_ticket = take(sizeof(uint32_t));
  L.off_pub = take(sizeof(unsigned long long) * L.nctas);
  L.off_comp = take(L.ncomp);
  L.off_diff = take(sizeof(int32_t) * L.nblocks);
  L.off_coef = take(sizeof(int16_t) * 64 * L.nblocks);
  L.off_plane = take(L.nplane);
  L.total = o;
  return L;
}

// the block a call copies in: S headers, then S jobs
size_t block_jobs_offset(int S) { return align256(sizeof(cp_jpeg_header) * S); }

// exclusive sum over a CTA of `kThreads`; *total gets the CTA's sum
template <int kThreads>
__device__ int64_t cta_exclusive(int64_t v, int64_t* total) {
  __shared__ int64_t warp_sum[kThreads / 32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int64_t x = v;
  for (int d = 1; d < 32; d <<= 1) {
    int64_t y = __shfl_up_sync(0xffffffffu, x, d);
    if (lane >= d) x += y;
  }
  if (lane == 31) warp_sum[w] = x;
  __syncthreads();
  if (w == 0) {
    int64_t s = lane < kThreads / 32 ? warp_sum[lane] : 0;
    for (int d = 1; d < 32; d <<= 1) {
      int64_t y = __shfl_up_sync(0xffffffffu, s, d);
      if (lane >= d) s += y;
    }
    if (lane < kThreads / 32) warp_sum[lane] = s;
  }
  __syncthreads();
  int64_t r = x - v + (w ? warp_sum[w - 1] : 0);
  *total = warp_sum[kThreads / 32 - 1];
  __syncthreads();
  return r;
}

// ---------------------------------------------------------------- 1. scan preparation
__global__ void __launch_bounds__(kPrepThreads) jpeg_prep(const Job* jobs, Seg* segs, const uint8_t* bytes,
                                                          uint8_t* comp, int words, int32_t* errors) {
  const int f = blockIdx.x, t = threadIdx.x;
  const Job& J = jobs[f];
  const uint8_t* r = bytes + J.raw;
  uint8_t* out = comp + J.comp;
  Seg* sg = segs + J.seg0;
  const int64_t n = J.nraw;
  const int nseg = J.nseg;
  for (int s = t; s < nseg; s += kPrepThreads) sg[s] = Seg{0, 0, 0, 0, f, s};
  __syncthreads();
  int64_t kept = 0, markers = 0;
  int err = 0;
  for (int64_t base = 0; base < n; base += 8 * kPrepThreads) {
    const int64_t i0 = base + 8 * (int64_t)t;
    int kc = 0, mc = 0;
    uint8_t c[10];
    for (int q = 0; q < 10; ++q) {
      int64_t i = i0 - 1 + q;
      c[q] = i >= 0 && i < n ? r[i] : 0;
    }
    uint32_t keep = 0, mark = 0;
    for (int q = 0; q < 8 && i0 + q < n; ++q) {
      uint8_t prev = c[q], v = c[q + 1], next = c[q + 2];
      if (v == 0xFF) {
        if (next == 0x00) keep |= 1u << q;
      } else if (prev == 0xFF) {
        if (v >= 0xD0 && v <= 0xD7) mark |= 1u << q;
      } else {
        keep |= 1u << q;
      }
    }
    kc = __popc(keep);
    mc = __popc(mark);
    int64_t ktot, mtot;
    int64_t kx = cta_exclusive<kPrepThreads>(kc, &ktot);
    int64_t mx = cta_exclusive<kPrepThreads>(mc, &mtot);
    int64_t p = kept + kx, m = markers + mx;
    for (int q = 0; q < 8; ++q) {
      if (keep >> q & 1) out[p++] = c[q + 1];
      if (mark >> q & 1) {
        if (m < nseg - 1) {
          sg[m].end = (uint32_t)p;
          sg[m + 1].begin = (uint32_t)p;
          if (c[q + 1] != 0xD0 + (m & 7)) err |= CP_JPEG_ERR_RESTART;
        } else if (m == nseg - 1) {
          sg[m].end = (uint32_t)p;
        }
        ++m;
      }
    }
    kept += ktot;
    markers += mtot;
  }
  if (err) atomicOr(errors + f, err);
  __syncthreads();
  if (t == 0) {
    if (markers < nseg - 1) atomicOr(errors + f, CP_JPEG_ERR_RESTART);
    if (markers < nseg) sg[markers].end = (uint32_t)kept;
  }
  __syncthreads();
  // each segment's subsequences, in order, from the frame's first slot
  const uint32_t S = 32u * words;
  int64_t carry = 0;
  for (int base = 0; base < nseg; base += kPrepThreads) {
    int s = base + t;
    int64_t ns = 0;
    if (s < nseg) {
      uint32_t bits = (sg[s].end - sg[s].begin) * 8u;
      ns = bits ? (bits + S - 1) / S : 1;
    }
    int64_t tot;
    int64_t x = cta_exclusive<kPrepThreads>(ns, &tot);
    if (s < nseg) {
      sg[s].first_sub = J.sub0 + carry + x;
      sg[s].nsub = (int32_t)ns;
    }
    carry += tot;
  }
}

// every slot: its segment (global index, -1 for an unused slot), its guessed start state, no blocks
__global__ void jpeg_subs(const Job* jobs, int B, const Seg* segs, int words, int64_t nsub, int32_t* sub_seg,
                          uint64_t* state, uint64_t* bnd, int32_t* cnt) {
  int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (j >= nsub) return;
  int lo = 0, hi = B - 1;
  while (lo < hi) {
    int mid = (lo + hi + 1) / 2;
    if (jobs[mid].sub0 <= j) lo = mid; else hi = mid - 1;
  }
  const Job& J = jobs[lo];
  int32_t id = -1;
  uint64_t st = 0;
  if (j < J.sub0 + J.nsub) {                 // past a frame's own count (a slot's capacity, a skipped slot): unused
    int a = 0, e = J.nseg - 1;
    while (a < e) {
      int mid = (a + e + 1) / 2;
      if (segs[J.seg0 + mid].first_sub <= j) a = mid; else e = mid - 1;
    }
    const Seg& s = segs[J.seg0 + a];
    if (j >= s.first_sub && j < s.first_sub + s.nsub) {
      id = J.seg0 + a;
      st = pack(State{(uint32_t)((j - s.first_sub) * 32 * words), 0, 0});
    }
  }
  sub_seg[j] = id;
  state[j] = st;
  bnd[j] = st;
  cnt[j] = 0;
}

// ---------------------------------------------------------------- 2. synchronisation
// One thread's subsequence j in a synchronisation pass: its segment (sid < 0: an unused slot), its index i in the
// segment, its start state st, its exit ex and the blocks it begins.
struct Lane {
  int sid;
  const cp_jpeg_header* h;
  const uint8_t* seg;
  uint32_t nbytes, stop;
  int64_t i;
  State st, ex;
  int dcs;
};

// The lane of subsequence j, walked once from its start state (state[j], or `first` for a thread that takes its
// predecessor CTA's exit); exits[t] gets its exit.
__device__ Lane lane_walk(const cp_jpeg_header* hs, const Job* jobs, const Seg* segs, const uint8_t* comp, int words,
                          int64_t nsub, const int32_t* sub_seg, const uint64_t* state, int64_t j, bool take_first,
                          uint64_t first, uint64_t* exits) {
  Lane l{j < nsub ? sub_seg[j] : -1, nullptr, nullptr, 0, 0, 0, State{0, 0, 0}, State{0, 0, 0}, 0};
  if (l.sid >= 0) {
    const Seg& s = segs[l.sid];
    l.h = hs + s.frame;
    l.seg = comp + jobs[s.frame].comp + s.begin;
    l.nbytes = s.end - s.begin;
    l.i = j - s.first_sub;
    l.stop = (uint32_t)((l.i + 1) * 32u * words);
    l.st = unpack(l.i > 0 && take_first ? first : state[j]);
    l.ex = walk(*l.h, l.seg, l.nbytes, l.st, l.stop, l.dcs);
  }
  exits[threadIdx.x] = pack(l.ex);
  return l;
}

// The intra-CTA loop: every thread past the first re-walks from its predecessor's exit until no exit changes.
__device__ void lane_settle(Lane& l, uint64_t* exits) {
  const int t = threadIdx.x;
  for (;;) {
    __syncthreads();
    bool moved = false;
    if (l.sid >= 0 && l.i > 0 && t > 0 && exits[t - 1] != pack(l.st)) {
      l.st = unpack(exits[t - 1]);
      moved = true;
    }
    __syncthreads();
    if (moved) {
      l.ex = walk(*l.h, l.seg, l.nbytes, l.st, l.stop, l.dcs);
      exits[t] = pack(l.ex);
    }
    if (!__syncthreads_or(moved)) break;
  }
}

// One round (cp_jpeg_decode): thread 0 of a CTA starts from the exit its predecessor CTA handed on in the last round.
__global__ void __launch_bounds__(kSyncThreads) jpeg_sync(const cp_jpeg_header* hs, const Job* jobs, const Seg* segs,
                                                          const uint8_t* comp, int words, int64_t nsub,
                                                          const int32_t* sub_seg, uint64_t* state,
                                                          const uint64_t* bnd_in, uint64_t* bnd_out, int32_t* cnt,
                                                          int32_t* changed) {
  __shared__ uint64_t exits[kSyncThreads];
  const int t = threadIdx.x;
  const int64_t j = blockIdx.x * (int64_t)kSyncThreads + t;
  Lane l = lane_walk(hs, jobs, segs, comp, words, nsub, sub_seg, state, j, t == 0, j < nsub ? bnd_in[j] : 0, exits);
  lane_settle(l, exits);
  if (l.sid < 0) return;
  state[j] = pack(l.st);
  cnt[j] = l.dcs;
  if (t == kSyncThreads - 1 && j + 1 < nsub && sub_seg[j + 1] == l.sid) {
    uint64_t e = pack(l.ex);
    bnd_out[j + 1] = e;
    if (e != bnd_in[j + 1]) *changed = 1;
  }
}

// The one-pass form (cp_jpeg_decode_slots_dev), in the style of decoupled look-back: a CTA takes its place in the chain
// from an atomic ticket, so it only waits on a CTA that has already started; it settles speculatively, then, when its
// first subsequence continues a segment, waits for its predecessor's final exit, re-walks from it until nothing moves
// and publishes its own last exit.  The chain hands on exact states, so every state is the sequential decoder's.
constexpr unsigned long long kPublished = 1ull << 63;      // a packed state fills the low 48 bits
constexpr long long kSyncWaitNs = 1000000000ll;             // CP_JPEG_ERR_SYNC after about a second

__device__ unsigned long long load_acquire(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

__device__ void store_release(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

__device__ long long global_ns() {
  long long v;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(v));
  return v;
}

__global__ void __launch_bounds__(kSyncThreads) jpeg_sync_chained(const cp_jpeg_header* hs, const Job* jobs,
                                                                  const Seg* segs, const uint8_t* comp, int words,
                                                                  int64_t nsub, const int32_t* sub_seg,
                                                                  uint64_t* state, int32_t* cnt, uint32_t* ticket,
                                                                  unsigned long long* published, int32_t* errors) {
  __shared__ uint64_t exits[kSyncThreads];
  __shared__ uint32_t order;
  const int t = threadIdx.x;
  if (t == 0) order = atomicAdd(ticket, 1u);
  __syncthreads();
  const int64_t b = order, j = b * kSyncThreads + t;
  Lane l = lane_walk(hs, jobs, segs, comp, words, nsub, sub_seg, state, j, false, 0, exits);
  lane_settle(l, exits);
  if (t == 0 && l.sid >= 0 && l.i > 0) {
    unsigned long long v = 0;
    const long long t0 = global_ns();
    for (unsigned ns = 32; !(v = load_acquire(published + b - 1));) {
      if (global_ns() - t0 > kSyncWaitNs) break;
      __nanosleep(ns);
      if (ns < 4096) ns *= 2;
    }
    if (!v) {
      atomicOr(errors + segs[l.sid].frame, CP_JPEG_ERR_SYNC);
    } else if ((v & ~kPublished) != pack(l.st)) {
      l.st = unpack(v & ~kPublished);
      l.ex = walk(*l.h, l.seg, l.nbytes, l.st, l.stop, l.dcs);
      exits[0] = pack(l.ex);
    }
  }
  lane_settle(l, exits);
  if (l.sid >= 0) {
    state[j] = pack(l.st);
    cnt[j] = l.dcs;
  }
  if (t == kSyncThreads - 1) store_release(published + b, pack(l.ex) | kPublished);
}

// ---------------------------------------------------------------- 3. blocks before each subsequence
// one CTA per frame: the exclusive prefix sum over its own subsequences (emit takes differences within a segment)
__global__ void __launch_bounds__(1024) jpeg_scan(const Job* jobs, const int32_t* cnt, int32_t* scan) {
  const Job& J = jobs[blockIdx.x];
  const int64_t n = J.nsub;
  int64_t carry = 0;
  for (int64_t base = 0; base < n; base += 1024) {
    int64_t j = base + threadIdx.x;
    int64_t v = j < n ? cnt[J.sub0 + j] : 0, tot;
    int64_t x = cta_exclusive<1024>(v, &tot);
    if (j < n) scan[J.sub0 + j] = (int32_t)(carry + x);
    carry += tot;
  }
}

// ---------------------------------------------------------------- 4. the final pass
__global__ void jpeg_emit(const cp_jpeg_header* hs, const Job* jobs, const Seg* segs, const uint8_t* comp, int words,
                          int64_t nsub, const int32_t* sub_seg, const uint64_t* state, const int32_t* scan,
                          int16_t* coef, int32_t* diff, int32_t* errors) {
  const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (j >= nsub || sub_seg[j] < 0) return;
  const Seg& s = segs[sub_seg[j]];
  const cp_jpeg_header& h = hs[s.frame];
  const Job& J = jobs[s.frame];
  const int64_t i = j - s.first_sub;
  const int64_t nmcu = (int64_t)h.mcux * h.mcuy, mcu0 = h.restart_interval ? (int64_t)s.index * h.restart_interval : 0;
  const int64_t mcus = h.restart_interval ? min((int64_t)h.restart_interval, nmcu - mcu0) : nmcu;
  const int64_t blk = J.blk0 + mcu0 * h.blocks_per_mcu;
  int err = emit(h, comp + J.comp + s.begin, s.end - s.begin, unpack(state[j]), (uint32_t)((i + 1) * 32 * words),
                 scan[j] - scan[s.first_sub], (int)(mcus * h.blocks_per_mcu), i == s.nsub - 1, coef + blk * 64,
                 diff + blk);
  if (err) atomicOr(errors + s.frame, err);
}

// ---------------------------------------------------------------- 5. DC prediction
__global__ void __launch_bounds__(1024) jpeg_dc(const cp_jpeg_header* hs, const Job* jobs, const int32_t* diff,
                                                int16_t* coef) {
  const cp_jpeg_header& h = hs[blockIdx.x];
  const int c = blockIdx.y;
  if (c >= h.ncomp) return;
  const int64_t blk0 = jobs[blockIdx.x].blk0;
  const int bpm = h.blocks_per_mcu;
  const int ny = h.ncomp == 1 ? 1 : h.comp_h[0] * h.comp_v[0];
  const int nb = c == 0 ? ny : 1, off = c == 0 ? 0 : ny + c - 1;
  const int64_t nmcu = (int64_t)h.mcux * h.mcuy, n = nmcu * nb;
  const int ri = h.restart_interval;
  const int64_t per = (n + 1023) / 1024, a = threadIdx.x * per, e = min(n, a + per);
  auto block_of = [&](int64_t q, bool& reset) {
    int64_t m = q / nb, kk = q % nb;
    reset = q == 0 || (ri && kk == 0 && m % ri == 0);
    return blk0 + m * bpm + off + kk;
  };
  bool flag = false;
  int32_t sum = 0;
  for (int64_t q = a; q < e; ++q) {
    bool rs;
    int64_t g = block_of(q, rs);
    if (rs) { flag = true; sum = 0; }
    sum += diff[g];
  }
  // segmented inclusive scan of (flag, sum) over the CTA
  __shared__ int32_t ss[1024];
  __shared__ uint8_t sf[1024];
  ss[threadIdx.x] = sum;
  sf[threadIdx.x] = flag;
  __syncthreads();
  for (int d = 1; d < 1024; d <<= 1) {
    int32_t ps = 0;
    bool pf = false;
    if (threadIdx.x >= d) { ps = ss[threadIdx.x - d]; pf = sf[threadIdx.x - d]; }
    __syncthreads();
    if (threadIdx.x >= d && !flag) { sum += ps; flag = pf; }
    ss[threadIdx.x] = sum;
    sf[threadIdx.x] = flag;
    __syncthreads();
  }
  int32_t acc = threadIdx.x ? ss[threadIdx.x - 1] : 0;
  for (int64_t q = a; q < e; ++q) {
    bool rs;
    int64_t g = block_of(q, rs);
    if (rs) acc = 0;
    acc += diff[g];
    coef[g * 64] = (int16_t)acc;
  }
}

// ---------------------------------------------------------------- 6. dequantisation and IDCT
__global__ void jpeg_idct(const cp_jpeg_header* hs, const Job* jobs, const int16_t* coef, uint8_t* planes) {
  const cp_jpeg_header& h = hs[blockIdx.y];
  const Job& J = jobs[blockIdx.y];
  const int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (g >= (int64_t)h.mcux * h.mcuy * h.blocks_per_mcu) return;
  int x, y;
  int c = block_origin(h, g, x, y);
  int ps = plane_w(h, c);
  idct_islow(coef + (J.blk0 + g) * 64, h.quant[c], planes + J.plane[c] + (int64_t)y * ps + x, ps);
}

// ---------------------------------------------------------------- 7. up-sampling, colour and orientation
__global__ void jpeg_color(const cp_jpeg_header* hs, const Job* jobs, const uint8_t* planes, uint8_t* bgr) {
  const cp_jpeg_header& h = hs[blockIdx.y];
  const Job& J = jobs[blockIdx.y];
  const int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (q >= (int64_t)h.out_h * h.out_w) return;
  const uint8_t* pl[3] = {planes + J.plane[0], planes + J.plane[1], planes + J.plane[2]};
  int ps[3] = {plane_w(h, 0), h.ncomp == 3 ? plane_w(h, 1) : 0, h.ncomp == 3 ? plane_w(h, 2) : 0};
  uint8_t v[3];
  pixel(h, pl, ps, (int)(q % h.out_w), (int)(q / h.out_w), v);
  uint8_t* o = bgr + J.out + q * 3;
  o[0] = v[0]; o[1] = v[1]; o[2] = v[2];
}

// ---------------------------------------------------------------- a corrupt slot detects nothing
// n_valid[m * n + r] = 0 for every category m of row r whose slot (rows[r], or r) has a nonzero error word
__global__ void jpeg_mask_counts(const int32_t* errors, const int32_t* rows, int n, int M, int32_t* n_valid) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n * M) return;
  const int r = q % n;
  if (errors[rows ? rows[r] : r]) n_valid[q] = 0;
}

thread_local int g_last_rounds = 0;

}  // namespace
}  // namespace jpeg
}  // namespace cp

using namespace cp::jpeg;

extern "C" int cp_jpeg_parse(const uint8_t* bytes, int64_t n, cp_jpeg_header* h) {
  if (!bytes || n < 0 || !h) return cp::fail(CP_ERR_INVALID, "cp_jpeg_parse: null or negative argument");
  int r = parse(bytes, n, h);
  if (r != CP_JPEG_OK) return cp::fail(CP_ERR_INVALID, "cp_jpeg_parse: refused, reason " + std::to_string(r));
  return 0;
}

static int check_headers(const char* who, const cp_jpeg_header* hs, int32_t B) {
  if (!hs || B <= 0) return cp::fail(CP_ERR_INVALID, std::string(who) + ": no headers");
  for (int b = 0; b < B; ++b) {
    const cp_jpeg_header& h = hs[b];
    if (h.status != CP_JPEG_OK || h.width <= 0 || h.height <= 0 || h.scan_end < h.scan_begin ||
        h.scan_end - h.scan_begin >= (int64_t)1 << 28)
      return cp::fail(CP_ERR_INVALID, std::string(who) + ": header " + std::to_string(b) + " is not a parsed, "
                      "supported JPEG (status " + std::to_string(h.status) + ")");
  }
  return 0;
}

extern "C" size_t cp_jpeg_workspace_bytes(const cp_jpeg_header* headers, int32_t B) {
  if (check_headers("cp_jpeg_workspace_bytes", headers, B)) return 0;
  return layout(headers, B, 1).total;
}

extern "C" int cp_jpeg_last_rounds(void) { return g_last_rounds; }

extern "C" int cp_jpeg_decode(const cp_jpeg_header* headers, int32_t B, const uint8_t* d_bytes,
                              const int64_t* byte_offsets, uint8_t* d_bgr, const int64_t* out_offsets, void* workspace,
                              size_t ws_bytes, int32_t* d_errors, int32_t subseq_words, void* stream) {
  const char* who = "cp_jpeg_decode";
  if (int rc = check_headers(who, headers, B)) return rc;
  if (!d_bytes || !byte_offsets || !d_bgr || !out_offsets || !workspace || !d_errors || subseq_words < 0)
    return cp::fail(CP_ERR_INVALID, "cp_jpeg_decode: null argument or negative subseq_words");
  const int words = subseq_words ? subseq_words : kDefaultSubseqWords;
  Layout L = layout(headers, B, words);
  if (ws_bytes < L.total)
    return cp::fail(CP_ERR_INVALID, "cp_jpeg_decode: workspace of " + std::to_string(ws_bytes) + " bytes, needs " +
                    std::to_string(L.total));
  for (int b = 0; b < B; ++b) {
    if (byte_offsets[b] < 0 || out_offsets[b] < 0)
      return cp::fail(CP_ERR_INVALID, "cp_jpeg_decode: negative offset of frame " + std::to_string(b));
    L.jobs[b].raw = byte_offsets[b] + headers[b].scan_begin;
    L.jobs[b].out = out_offsets[b];
  }
  cudaStream_t s = (cudaStream_t)stream;
  uint8_t* ws = (uint8_t*)workspace;
  cp_jpeg_header* d_hdr = (cp_jpeg_header*)(ws + L.off_hdr);
  Job* d_job = (Job*)(ws + L.off_job);
  Seg* d_seg = (Seg*)(ws + L.off_seg);
  int32_t* d_subseg = (int32_t*)(ws + L.off_subseg);
  uint64_t* d_state = (uint64_t*)(ws + L.off_state);
  uint64_t* d_bnd = (uint64_t*)(ws + L.off_bnd);
  int32_t* d_cnt = (int32_t*)(ws + L.off_cnt);
  int32_t* d_scan = (int32_t*)(ws + L.off_scan);
  int32_t* d_flag = (int32_t*)(ws + L.off_flag);
  uint8_t* d_comp = ws + L.off_comp;
  int32_t* d_diff = (int32_t*)(ws + L.off_diff);
  int16_t* d_coef = (int16_t*)(ws + L.off_coef);
  uint8_t* d_plane = ws + L.off_plane;

  CP_CUDA_CHECK(cudaMemcpyAsync(d_hdr, headers, sizeof(cp_jpeg_header) * B, cudaMemcpyHostToDevice, s));
  CP_CUDA_CHECK(cudaMemcpyAsync(d_job, L.jobs.data(), sizeof(Job) * B, cudaMemcpyHostToDevice, s));
  CP_CUDA_CHECK(cudaMemsetAsync(d_errors, 0, sizeof(int32_t) * B, s));
  CP_CUDA_CHECK(cudaMemsetAsync(d_diff, 0, sizeof(int32_t) * L.nblocks, s));
  CP_CUDA_CHECK(cudaMemsetAsync(d_coef, 0, sizeof(int16_t) * 64 * L.nblocks, s));

  jpeg_prep<<<B, kPrepThreads, 0, s>>>(d_job, d_seg, d_bytes, d_comp, words, d_errors);
  CP_LAUNCH_CHECK("jpeg_prep");
  const unsigned gsub = (unsigned)((L.nsub + 255) / 256);
  jpeg_subs<<<gsub, 256, 0, s>>>(d_job, B, d_seg, words, L.nsub, d_subseg, d_state, d_bnd, d_cnt);
  CP_LAUNCH_CHECK("jpeg_subs");
  // the host repeats the round while a CTA handed a changed state to the next one
  int rounds = 0;
  for (int32_t moved = 1; moved; ++rounds) {
    const uint64_t* bin = d_bnd + (rounds & 1) * L.nsub;
    uint64_t* bout = d_bnd + ((rounds + 1) & 1) * L.nsub;
    CP_CUDA_CHECK(cudaMemcpyAsync(bout, bin, sizeof(uint64_t) * L.nsub, cudaMemcpyDeviceToDevice, s));
    CP_CUDA_CHECK(cudaMemsetAsync(d_flag, 0, sizeof(int32_t), s));
    jpeg_sync<<<(unsigned)((L.nsub + kSyncThreads - 1) / kSyncThreads), kSyncThreads, 0, s>>>(
        d_hdr, d_job, d_seg, d_comp, words, L.nsub, d_subseg, d_state, bin, bout, d_cnt, d_flag);
    CP_LAUNCH_CHECK("jpeg_sync");
    CP_CUDA_CHECK(cudaMemcpyAsync(&moved, d_flag, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    CP_CUDA_CHECK(cudaStreamSynchronize(s));
  }
  g_last_rounds = rounds;
  jpeg_scan<<<B, 1024, 0, s>>>(d_job, d_cnt, d_scan);
  CP_LAUNCH_CHECK("jpeg_scan");
  jpeg_emit<<<gsub, 256, 0, s>>>(d_hdr, d_job, d_seg, d_comp, words, L.nsub, d_subseg, d_state, d_scan, d_coef, d_diff,
                                 d_errors);
  CP_LAUNCH_CHECK("jpeg_emit");
  jpeg_dc<<<dim3(B, 3), 1024, 0, s>>>(d_hdr, d_job, d_diff, d_coef);
  CP_LAUNCH_CHECK("jpeg_dc");
  jpeg_idct<<<dim3((unsigned)((L.maxblocks + 127) / 128), B), 128, 0, s>>>(d_hdr, d_job, d_coef, d_plane);
  CP_LAUNCH_CHECK("jpeg_idct");
  jpeg_color<<<dim3((unsigned)((L.maxpix + 255) / 256), B), 256, 0, s>>>(d_hdr, d_job, d_plane, d_bgr);
  CP_LAUNCH_CHECK("jpeg_color");
  return 0;
}

static int check_slots(const char* who, int32_t S, const int32_t* hw, const int64_t* max_bytes, int32_t subseq_words) {
  if (S <= 0 || !hw || !max_bytes || subseq_words < 0)
    return cp::fail(CP_ERR_INVALID, std::string(who) + ": no slots, null sizes or negative subseq_words");
  for (int s = 0; s < S; ++s)
    if (hw[2 * s] <= 0 || hw[2 * s + 1] <= 0 || (int64_t)hw[2 * s] * hw[2 * s + 1] > ((int64_t)1 << 30) ||
        max_bytes[s] <= 0 || max_bytes[s] >= ((int64_t)1 << 28))
      return cp::fail(CP_ERR_INVALID, std::string(who) + ": slot " + std::to_string(s) + " needs a decoded size of "
                      "1 to 2^30 pixels and 1 <= max_bytes < 2^28");
  return 0;
}

extern "C" size_t cp_jpeg_slots_workspace_bytes(int32_t S, const int32_t* hw, const int64_t* max_bytes,
                                               int32_t subseq_words) {
  if (check_slots("cp_jpeg_slots_workspace_bytes", S, hw, max_bytes, subseq_words)) return 0;
  return slot_layout(S, hw, max_bytes, subseq_words ? subseq_words : kDefaultSubseqWords).total;
}

extern "C" size_t cp_jpeg_slots_block_bytes(int32_t S) {
  if (S <= 0) return 0;
  return block_jobs_offset(S) + sizeof(Job) * S;
}

extern "C" int cp_jpeg_slots_prepare(int32_t S, const int32_t* hw, const int64_t* max_bytes, int32_t subseq_words,
                                     const cp_jpeg_header* headers, const int64_t* nbytes, const int64_t* out_offsets,
                                     void* host_block) {
  const char* who = "cp_jpeg_slots_prepare";
  if (int rc = check_slots(who, S, hw, max_bytes, subseq_words)) return rc;
  if (!headers || !nbytes || !out_offsets || !host_block)
    return cp::fail(CP_ERR_INVALID, "cp_jpeg_slots_prepare: null argument");
  const int words = subseq_words ? subseq_words : kDefaultSubseqWords;
  for (int s = 0; s < S; ++s) {
    if (nbytes[s] == 0) continue;
    const cp_jpeg_header& h = headers[s];
    const std::string slot = std::string(who) + ": slot " + std::to_string(s);
    if (check_headers(slot.c_str(), &h, 1)) return CP_ERR_INVALID;
    if (h.out_h != hw[2 * s] || h.out_w != hw[2 * s + 1])
      return cp::fail(CP_ERR_INVALID, slot + " decodes to " + std::to_string(h.out_h) + " x " +
                      std::to_string(h.out_w) + ", the slot is " + std::to_string(hw[2 * s]) + " x " +
                      std::to_string(hw[2 * s + 1]));
    if (nbytes[s] < 0 || nbytes[s] > max_bytes[s] || h.scan_end > nbytes[s])
      return cp::fail(CP_ERR_INVALID, slot + ": " + std::to_string(nbytes[s]) + " bytes (scan to " +
                      std::to_string(h.scan_end) + "), the slot takes at most " + std::to_string(max_bytes[s]));
    if (out_offsets[s] < 0) return cp::fail(CP_ERR_INVALID, slot + ": negative output offset");
  }
  SlotLayout L = slot_layout(S, hw, max_bytes, words);
  uint8_t* blk = (uint8_t*)host_block;
  cp_jpeg_header* hb = (cp_jpeg_header*)blk;
  Job* jb = (Job*)(blk + block_jobs_offset(S));
  memset(blk, 0, cp_jpeg_slots_block_bytes(S));
  for (int s = 0; s < S; ++s) {
    Job j = L.base[s];                           // a skipped slot: its regions, no segment, no subsequence
    if (nbytes[s]) {
      const cp_jpeg_header& h = headers[s];
      hb[s] = h;
      j.raw += h.scan_begin;
      j.nraw = h.scan_end - h.scan_begin;
      const SlotCap need = frame_need(h, words);
      j.nseg = (int32_t)need.nseg;
      j.nsub = need.nsub;
      int64_t p = j.plane[0];
      for (int c = 0; c < 3; ++c) {
        j.plane[c] = p;
        if (c < h.ncomp) p += (int64_t)plane_w(h, c) * plane_h(h, c);
      }
      j.out = out_offsets[s];
    }
    jb[s] = j;
  }
  return 0;
}

extern "C" int cp_jpeg_decode_slots_dev(const void* d_block, int32_t S, const int32_t* hw, const int64_t* max_bytes,
                                        int32_t subseq_words, const uint8_t* d_bytes, uint8_t* d_bgr, void* workspace,
                                        size_t ws_bytes, int32_t* d_errors, void* stream) {
  const char* who = "cp_jpeg_decode_slots_dev";
  if (int rc = check_slots(who, S, hw, max_bytes, subseq_words)) return rc;
  if (!d_block || !d_bytes || !d_bgr || !workspace || !d_errors)
    return cp::fail(CP_ERR_INVALID, "cp_jpeg_decode_slots_dev: null argument");
  const int words = subseq_words ? subseq_words : kDefaultSubseqWords;
  SlotLayout L = slot_layout(S, hw, max_bytes, words);
  if (ws_bytes < L.total)
    return cp::fail(CP_ERR_INVALID, "cp_jpeg_decode_slots_dev: workspace of " + std::to_string(ws_bytes) +
                    " bytes, needs " + std::to_string(L.total));
  cudaStream_t s = (cudaStream_t)stream;
  uint8_t* ws = (uint8_t*)workspace;
  const cp_jpeg_header* d_hdr = (const cp_jpeg_header*)d_block;
  const Job* d_job = (const Job*)((const uint8_t*)d_block + block_jobs_offset(S));
  Seg* d_seg = (Seg*)(ws + L.off_seg);
  int32_t* d_subseg = (int32_t*)(ws + L.off_subseg);
  uint64_t* d_state = (uint64_t*)(ws + L.off_state);
  int32_t* d_cnt = (int32_t*)(ws + L.off_cnt);
  int32_t* d_scan = (int32_t*)(ws + L.off_scan);
  uint32_t* d_ticket = (uint32_t*)(ws + L.off_ticket);
  unsigned long long* d_pub = (unsigned long long*)(ws + L.off_pub);
  uint8_t* d_comp = ws + L.off_comp;
  int32_t* d_diff = (int32_t*)(ws + L.off_diff);
  int16_t* d_coef = (int16_t*)(ws + L.off_coef);
  uint8_t* d_plane = ws + L.off_plane;

  // the ticket and the published exits are contiguous: one memset resets the chain
  CP_CUDA_CHECK(cudaMemsetAsync(d_ticket, 0, L.off_comp - L.off_ticket, s));
  CP_CUDA_CHECK(cudaMemsetAsync(d_errors, 0, sizeof(int32_t) * S, s));
  CP_CUDA_CHECK(cudaMemsetAsync(d_diff, 0, sizeof(int32_t) * L.nblocks, s));
  CP_CUDA_CHECK(cudaMemsetAsync(d_coef, 0, sizeof(int16_t) * 64 * L.nblocks, s));
  jpeg_prep<<<S, kPrepThreads, 0, s>>>(d_job, d_seg, d_bytes, d_comp, words, d_errors);
  CP_LAUNCH_CHECK("jpeg_prep");
  const unsigned gsub = (unsigned)((L.nsub + 255) / 256);
  jpeg_subs<<<gsub, 256, 0, s>>>(d_job, S, d_seg, words, L.nsub, d_subseg, d_state, d_state, d_cnt);
  CP_LAUNCH_CHECK("jpeg_subs");
  jpeg_sync_chained<<<(unsigned)L.nctas, kSyncThreads, 0, s>>>(d_hdr, d_job, d_seg, d_comp, words, L.nsub, d_subseg,
                                                               d_state, d_cnt, d_ticket, d_pub, d_errors);
  CP_LAUNCH_CHECK("jpeg_sync_chained");
  jpeg_scan<<<S, 1024, 0, s>>>(d_job, d_cnt, d_scan);
  CP_LAUNCH_CHECK("jpeg_scan");
  jpeg_emit<<<gsub, 256, 0, s>>>(d_hdr, d_job, d_seg, d_comp, words, L.nsub, d_subseg, d_state, d_scan, d_coef, d_diff,
                                 d_errors);
  CP_LAUNCH_CHECK("jpeg_emit");
  jpeg_dc<<<dim3(S, 3), 1024, 0, s>>>(d_hdr, d_job, d_diff, d_coef);
  CP_LAUNCH_CHECK("jpeg_dc");
  jpeg_idct<<<dim3((unsigned)((L.maxblocks + 127) / 128), S), 128, 0, s>>>(d_hdr, d_job, d_coef, d_plane);
  CP_LAUNCH_CHECK("jpeg_idct");
  jpeg_color<<<dim3((unsigned)((L.maxpix + 255) / 256), S), 256, 0, s>>>(d_hdr, d_job, d_plane, d_bgr);
  CP_LAUNCH_CHECK("jpeg_color");
  return 0;
}

extern "C" int cp_jpeg_mask_counts_dev(const int32_t* d_errors, const int32_t* d_rows, int32_t n, int32_t M,
                                       int32_t* d_n_valid, void* stream) {
  if (!d_errors || !d_n_valid || n <= 0 || M <= 0)
    return cp::fail(CP_ERR_INVALID, "cp_jpeg_mask_counts_dev: null buffer or no rows");
  const int q = n * M;
  jpeg_mask_counts<<<(q + 255) / 256, 256, 0, (cudaStream_t)stream>>>(d_errors, d_rows, n, M, d_n_valid);
  CP_LAUNCH_CHECK("jpeg_mask_counts");
  return 0;
}
