// b200_hevc_syntax.h -- HEVC slice-data decoding (CABAC 9.3 + coding-quadtree syntax 7.3.8 + intra-mode 8.4.2 and
// QP 8.6.1 derivation) as ONE piece of source compiled for both the host front-end (b200_hevc_parse.cc) and the
// device entropy-decoding kernel (b200_hevc_entropy.cu).  One instance decodes one CABAC sub-stream: a slice segment,
// or -- with entropy_coding_sync (WPP) -- one CTB row of it; sub-streams of a picture run concurrently on the GPU as a
// wavefront (context hand-over after the 2nd CTB of the row above, 9.3.2.2), sequentially on the host.
// Output = the command stream of b200_hevc_types.h.  No pixel is touched here.
#pragma once
#include <cassert>
#include <cstdint>
#include <cstring>
#include "b200_hevc_types.h"

#if defined(__CUDA_ARCH__) && !defined(B200_SYNTAX_HOST_ONLY)
#define B200_SYN_DEVICE 1
#endif
#if defined(__CUDACC__) && !defined(B200_SYNTAX_HOST_ONLY)
// B200_HDN: one out-of-line copy per function on the device.  Full inlining of the syntax tree blew the entropy kernel
// up to 38k SASS instructions (0.6 MB): the instruction cache, not arithmetic, set the pace of the lone decoding lane.
#define B200_HDN __host__ __device__ __noinline__
#define B200_NOUNROLL _Pragma("unroll 1")
#define B200_HD __host__ __device__
#define B200_HDI __host__ __device__ __forceinline__
#define B200_TABLE(type, name, dims, ...) static const type h_##name dims = __VA_ARGS__; static __device__ const type d_##name dims = __VA_ARGS__;
#else
#define B200_HDN
#define B200_NOUNROLL
#define B200_HD
#define B200_HDI inline
#define B200_TABLE(type, name, dims, ...) static const type h_##name dims = __VA_ARGS__;
#endif
#if defined(B200_SYN_DEVICE) && !defined(B200_T)
#define B200_T(name) d_##name
#endif
#ifdef B200_SYN_DEVICE
// data written by ANOTHER sub-stream's thread (possibly on another SM): bypass the non-coherent L1
#define B200_LD_SHARED(p) __ldcg(p)
#else
#ifndef B200_T
#define B200_T(name) h_##name
#endif
#define B200_LD_SHARED(p) (*(p))
#endif

namespace b200 {
namespace syn {

// Context states and the hot lookup tables live in SHARED memory on the device.  Going through generic pointers costs a
// 64-bit address, descriptor moves and a slower generic load per access (measured: 72 SASS instructions per
// sig_coeff_flag); these handles are 32-bit shared-window addresses there and plain pointers on the host.
#ifdef B200_SYN_DEVICE
typedef uint32_t CtxPtr;
typedef uint32_t TabPtr;
struct U2 { uint32_t x, y; };
// No "memory" clobbers: the context array is only ever touched through these handles, and asm volatile statements keep
// their program order among themselves (loads of one context never pass stores to it).
__device__ __forceinline__ U2 ctx_ld(CtxPtr p) { U2 v; asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(p)); return v; }
__device__ __forceinline__ void ctx_st(CtxPtr p, U2 v) { asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(p), "r"(v.x), "r"(v.y)); }
__device__ __forceinline__ CtxPtr ctx_at(CtxPtr base, int i) { return base + 8u * (uint32_t)i; }
__device__ __forceinline__ uint32_t tab_ld8(TabPtr p, int i) { uint32_t v; asm("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(p + (uint32_t)i)); return v; }
__device__ __forceinline__ U2 tab_ld64(TabPtr p, int i) { U2 v; asm("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(p + 8u * (uint32_t)i)); return v; }
__device__ __forceinline__ uint32_t tab_ld32(TabPtr p, int i) { uint32_t v; asm("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(p + 4u * (uint32_t)i)); return v; }
#define B200_TADDR(name) ((::b200::syn::TabPtr)__cvta_generic_to_shared(&B200_T(name)))
#else
struct U2 { uint32_t x, y; };
typedef U2* CtxPtr;
typedef const uint8_t* TabPtr;
inline U2 ctx_ld(CtxPtr p) { return *p; }
inline void ctx_st(CtxPtr p, U2 v) { *p = v; }
inline CtxPtr ctx_at(CtxPtr base, int i) { return base + i; }
inline uint32_t tab_ld8(TabPtr p, int i) { return p[i]; }
inline uint32_t tab_ld32(TabPtr p, int i) { uint32_t v; memcpy(&v, p + 4 * (size_t)i, 4); return v; }
inline U2 tab_ld64(TabPtr p, int i) { uint64_t v; memcpy(&v, p + 8 * (size_t)i, 8); return U2{(uint32_t)v, (uint32_t)(v >> 32)}; }
#define B200_TADDR(name) (reinterpret_cast<::b200::syn::TabPtr>(&B200_T(name)))
#endif

enum { CTX_SAO_MERGE = 0, CTX_SAO_TYPE = 1, CTX_SPLIT_CU = 2, CTX_PART_MODE = 5, CTX_PREV_INTRA = 6,
       CTX_CHROMA_PRED = 7, CTX_SPLIT_TR = 8, CTX_CBF_LUMA = 11, CTX_CBF_CHROMA = 13, CTX_QP_DELTA = 18,
       CTX_TSKIP = 20, CTX_LAST_X = 22, CTX_LAST_Y = 40, CTX_CSBF = 58, CTX_SIG = 62, CTX_GT1 = 104,
       CTX_GT2 = 128, CTX_TQ_BYPASS = 134, CTX_COUNT = 135, CTX_STRIDE = 144,
       CTX_SCRATCH = 8 };   // device: 8-byte slots behind the context array = the 16 level words of residual_coding's emission

// Tables 9-5 .. 9-37, initType 0 (I slices)
B200_TABLE(uint8_t, kInitI, [CTX_COUNT], {
  153, 200, 139, 141, 157, 184, 184, 63, 153, 138, 138, 111, 141, 94, 138, 182, 154, 154, 154, 154, 139, 139,
  110, 110, 124, 125, 140, 153, 125, 127, 140, 109, 111, 143, 127, 111, 79, 108, 123, 63,
  110, 110, 124, 125, 140, 153, 125, 127, 140, 109, 111, 143, 127, 111, 79, 108, 123, 63,
  91, 171, 134, 141,
  111, 111, 125, 110, 110, 94, 124, 108, 124, 107, 125, 141, 179, 153, 125, 107, 125, 141, 179, 153, 125,
  107, 125, 141, 179, 153, 125, 140, 139, 182, 182, 152, 136, 152, 136, 153, 136, 139, 111, 136, 139, 111,
  140, 92, 137, 138, 140, 152, 138, 139, 153, 74, 149, 92, 139, 107, 122, 152, 140, 179, 166, 182, 140, 227, 122, 197,
  138, 153, 136, 167, 152, 152,
  154})
// Table 9-46 (rangeTabLps) and 9-47 (transIdxLps)
B200_TABLE(uint32_t, kLps4, [64], {0xf0d0b080u, 0xe3c5a780u, 0xd8bb9e80u, 0xcdb2967bu, 0xc3a98e74u, 0xb9a0876fu, 0xaf988069u, 0xa6907a64u, 0x9e89745fu, 0x96826e5au, 0x8e7b6855u, 0x87756351u, 0x806f5e4du, 0x7a695949u, 0x74645545u, 0x6e5f5042u, 0x685a4c3eu, 0x6356483bu, 0x5e514538u, 0x594d4135u, 0x55493e33u, 0x50453b30u, 0x4c42382eu, 0x483f352bu, 0x453b3229u, 0x41383027u, 0x3e362d25u, 0x3b332b23u, 0x38302921u, 0x352e2720u, 0x322b251eu, 0x3029231du, 0x2d27211bu, 0x2b251f1au, 0x29231e18u, 0x27211c17u, 0x25201b16u, 0x231e1a15u, 0x211d1814u, 0x1f1b1713u, 0x1e1a1612u, 0x1c191511u, 0x1b171410u, 0x1916130fu, 0x1815120eu, 0x1714110eu, 0x1613100du, 0x15120f0cu, 0x14110e0cu, 0x13100e0bu, 0x120f0d0bu, 0x110f0c0au, 0x100e0c0au, 0x0f0d0b09u, 0x0e0c0b09u, 0x0e0c0a08u, 0x0d0b0908u, 0x0c0b0907u, 0x0c0a0907u, 0x0b0a0807u, 0x0b090806u, 0x0a090706u, 0x09080706u, 0x02020202u})   // rangeTabLps[state][0..3] packed little-endian
B200_TABLE(uint8_t, kTransLps, [64], {0,0,1,2,2,4,4,5,6,7,8,9,9,11,11,12,13,13,15,15,16,16,18,18,19,19,21,21,22,22,23,24,
  24,25,26,26,27,27,28,29,29,30,30,30,31,32,32,33,33,33,34,34,35,35,35,36,36,36,37,37,37,38,38,63})
B200_TABLE(uint8_t, kSigMap4, [16], {0, 1, 4, 5, 2, 3, 4, 5, 6, 6, 8, 8, 7, 7, 8, 8})
B200_TABLE(uint8_t, kChromaTab, [4], {0, 26, 10, 1})
// scan orders 6.5.3-6.5.5: [log2 block size 0..3][diagonal, horizontal, vertical][position] -> x / y
B200_TABLE(uint8_t, kScanX, [4][3][64], {{{0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0},{0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0},{0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0}},{{0,0,1,1,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0},{0,1,0,1,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0},{0,0,1,1,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0}},{{0,0,1,0,1,2,0,1,2,3,1,2,3,2,3,3,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0},{0,1,2,3,0,1,2,3,0,1,2,3,0,1,2,3,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0},{0,0,0,0,1,1,1,1,2,2,2,2,3,3,3,3,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0}},{{0,0,1,0,1,2,0,1,2,3,0,1,2,3,4,0,1,2,3,4,5,0,1,2,3,4,5,6,0,1,2,3,4,5,6,7,1,2,3,4,5,6,7,2,3,4,5,6,7,3,4,5,6,7,4,5,6,7,5,6,7,6,7,7},{0,1,2,3,4,5,6,7,0,1,2,3,4,5,6,7,0,1,2,3,4,5,6,7,0,1,2,3,4,5,6,7,0,1,2,3,4,5,6,7,0,1,2,3,4,5,6,7,0,1,2,3,4,5,6,7,0,1,2,3,4,5,6,7},{0,0,0,0,0,0,0,0,1,1,1,1,1,1,1,1,2,2,2,2,2,2,2,2,3,3,3,3,3,3,3,3,4,4,4,4,4,4,4,4,5,5,5,5,5,5,5,5,6,6,6,6,6,6,6,6,7,7,7,7,7,7,7,7}}})
B200_TABLE(uint8_t, kScanY, [4][3][64], {{{0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0},{0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0},{0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0}},{{0,1,0,1,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0},{0,0,1,1,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0},{0,1,0,1,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0}},{{0,1,0,2,1,0,3,2,1,0,3,2,1,3,2,3,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0},{0,0,0,0,1,1,1,1,2,2,2,2,3,3,3,3,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0},{0,1,2,3,0,1,2,3,0,1,2,3,0,1,2,3,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0}},{{0,1,0,2,1,0,3,2,1,0,4,3,2,1,0,5,4,3,2,1,0,6,5,4,3,2,1,0,7,6,5,4,3,2,1,0,7,6,5,4,3,2,1,7,6,5,4,3,2,7,6,5,4,3,7,6,5,4,7,6,5,7,6,7},{0,0,0,0,0,0,0,0,1,1,1,1,1,1,1,1,2,2,2,2,2,2,2,2,3,3,3,3,3,3,3,3,4,4,4,4,4,4,4,4,5,5,5,5,5,5,5,5,6,6,6,6,6,6,6,6,7,7,7,7,7,7,7,7},{0,1,2,3,4,5,6,7,0,1,2,3,4,5,6,7,0,1,2,3,4,5,6,7,0,1,2,3,4,5,6,7,0,1,2,3,4,5,6,7,0,1,2,3,4,5,6,7,0,1,2,3,4,5,6,7,0,1,2,3,4,5,6,7}}})

// derived from the scans above: 4x4 position (y << 2 | x) of scan index k and its inverse; sub-block scan index of (ys * 8 + xs);
// sig_coeff_flag context increments (9.3.4.2.5) per scan index: kSigCtx4 for 4x4 blocks, kSigCtxN[scan][prevCsbf] for larger ones
B200_TABLE(uint8_t, kScanPos, [3][16], {{0,4,1,8,5,2,12,9,6,3,13,10,7,14,11,15},{0,1,2,3,4,5,6,7,8,9,10,11,12,13,14,15},{0,4,8,12,1,5,9,13,2,6,10,14,3,7,11,15}})
B200_TABLE(uint8_t, kScanInv, [3][16], {{0,2,5,9,1,4,8,12,3,7,11,14,6,10,13,15},{0,1,2,3,4,5,6,7,8,9,10,11,12,13,14,15},{0,4,8,12,1,5,9,13,2,6,10,14,3,7,11,15}})
B200_TABLE(uint8_t, kSbInv, [4][3][64], {{{0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0},{0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0},{0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0}},{{0,2,0,0,0,0,0,0,1,3,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0},{0,1,0,0,0,0,0,0,2,3,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0},{0,2,0,0,0,0,0,0,1,3,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0}},{{0,2,5,9,0,0,0,0,1,4,8,12,0,0,0,0,3,7,11,14,0,0,0,0,6,10,13,15,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0},{0,1,2,3,0,0,0,0,4,5,6,7,0,0,0,0,8,9,10,11,0,0,0,0,12,13,14,15,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0},{0,4,8,12,0,0,0,0,1,5,9,13,0,0,0,0,2,6,10,14,0,0,0,0,3,7,11,15,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0}},{{0,2,5,9,14,20,27,35,1,4,8,13,19,26,34,42,3,7,12,18,25,33,41,48,6,11,17,24,32,40,47,53,10,16,23,31,39,46,52,57,15,22,30,38,45,51,56,60,21,29,37,44,50,55,59,62,28,36,43,49,54,58,61,63},{0,1,2,3,4,5,6,7,8,9,10,11,12,13,14,15,16,17,18,19,20,21,22,23,24,25,26,27,28,29,30,31,32,33,34,35,36,37,38,39,40,41,42,43,44,45,46,47,48,49,50,51,52,53,54,55,56,57,58,59,60,61,62,63},{0,8,16,24,32,40,48,56,1,9,17,25,33,41,49,57,2,10,18,26,34,42,50,58,3,11,19,27,35,43,51,59,4,12,20,28,36,44,52,60,5,13,21,29,37,45,53,61,6,14,22,30,38,46,54,62,7,15,23,31,39,47,55,63}}})
B200_TABLE(uint8_t, kSigCtx4, [3][16], {{0,2,1,6,3,4,7,6,4,5,7,8,5,8,8,8},{0,1,4,5,2,3,4,5,6,6,8,8,7,7,8,8},{0,2,6,7,1,3,6,7,4,4,8,8,5,5,8,8}})
B200_TABLE(uint8_t, kSigCtxN, [3][4][16], {{{2,1,1,1,1,1,0,0,0,0,0,0,0,0,0,0},{2,1,2,0,1,2,0,0,1,2,0,0,1,0,0,0},{2,2,1,2,1,0,2,1,0,0,1,0,0,0,0,0},{2,2,2,2,2,2,2,2,2,2,2,2,2,2,2,2}},{{2,1,1,0,1,1,0,0,1,0,0,0,0,0,0,0},{2,2,2,2,1,1,1,1,0,0,0,0,0,0,0,0},{2,1,0,0,2,1,0,0,2,1,0,0,2,1,0,0},{2,2,2,2,2,2,2,2,2,2,2,2,2,2,2,2}},{{2,1,1,0,1,1,0,0,1,0,0,0,0,0,0,0},{2,1,0,0,2,1,0,0,2,1,0,0,2,1,0,0},{2,2,2,2,1,1,1,1,0,0,0,0,0,0,0,0},{2,2,2,2,2,2,2,2,2,2,2,2,2,2,2,2}}})

B200_HD inline int clip3(int lo, int hi, int v) { return v < lo ? lo : (v > hi ? hi : v); }
B200_HD inline int imin(int a, int b) { return a < b ? a : b; }
#ifdef B200_SYN_DEVICE
B200_HD inline int hi_bit(uint32_t v) { return 31 - __clz((int)v); }          // v != 0
B200_HD inline int lo_bit(uint32_t v) { return __ffs((int)v) - 1; }
B200_HD inline int pop_count(uint32_t v) { return __popc(v); }
#else
B200_HD inline int hi_bit(uint32_t v) { return 31 - __builtin_clz(v); }
B200_HD inline int lo_bit(uint32_t v) { return __builtin_ctz(v); }
B200_HD inline int pop_count(uint32_t v) { return __builtin_popcount(v); }
#endif

// Warp-wide decoding on the device: all 32 lanes of a decoder warp run the (serial) syntax decoder on identical data, so
// every branch outside the lane-parallel sections is warp-uniform and a warp instruction costs one issue slot as before.
// The per-cell, per-context and per-coefficient work around the bins is split over the lanes in lane-parallel sections:
//   B200_LANES_BEGIN(); B200_LANE_FOR(k, n) { ... item k ... } B200_LANES_END();
// On the host the same source is a plain serial loop.  A section's stores (global map cells, shared contexts / scratch)
// are ordered before anything any lane does after B200_LANES_END.
#ifdef __CUDACC__
// volatile: read where it is needed instead of being kept live across the call chain
__device__ __forceinline__ int lane_id() { unsigned l; asm volatile("mov.u32 %0, %%laneid;" : "=r"(l)); return (int)l; }
// volatile asm with a memory clobber: also keeps its place among the (volatile asm) context loads and stores
__device__ __forceinline__ void warp_sync() { asm volatile("bar.warp.sync -1;" ::: "memory"); }
#endif
#ifdef B200_SYN_DEVICE
#ifdef B200_ENTROPY_CHECK_CONVERGENCE     // debug builds: every lane-parallel section is entered by the whole warp
#define B200_LANES_BEGIN() assert(__activemask() == 0xffffffffu)
#else
#define B200_LANES_BEGIN() ((void)0)
#endif
#define B200_LANE_FOR(k, n) B200_NOUNROLL for (int k = ::b200::syn::lane_id(); k < (n); k += 32)
#define B200_LANES_END() ::b200::syn::warp_sync()
#else
#define B200_LANES_BEGIN() ((void)0)
#define B200_LANE_FOR(k, n) B200_NOUNROLL for (int k = 0; k < (n); k++)
#define B200_LANES_END() ((void)0)
#endif

// Sequence / picture level parameters the slice data depends on (filled by the host from SPS + PPS).
struct SeqParams {
  int32_t W, H, log2ctb, wctb, hctb, w4, w8, h8, chroma, bd;
  int32_t log2_min_cb, log2_min_tb, log2_max_tb, max_th_depth_intra;
  int32_t sao_enabled, transform_skip, cu_qp_delta, qg_log2, sign_hiding, wpp, sao_scale_luma, sao_scale_chroma;
  int32_t dense;                 // 1: outputs appended densely (host, sequential); 0: fixed per-CTB slots (device, concurrent)
  int32_t tu_slots, coef_slots;  // per-CTB capacity when !dense
  int32_t pcm, pcm_bd_y, pcm_bd_c, pcm_shift_y, pcm_shift_c, log2_min_pcm, log2_max_pcm, pcm_lf_disabled;   // 7.4.3.2.1 (shift = BitDepth - PcmBitDepth)
  int32_t tq_bypass;             // transquant_bypass_enabled_flag
  int32_t tiles;                 // tiles_enabled_flag: sub-streams walk their tile's CTB rectangle; no per-row progress hand-shake
};

// One CABAC sub-stream.
struct Substream {
  uint32_t pic;                  // picture (tile) index in the batch
  uint32_t byte_begin, byte_end; // inside the picture's RBSP buffer (byte_begin need not be aligned)
  uint32_t ctb_begin, ctb_end;   // raster address of the first CTB; ctb_end - ctb_begin = number of CTBs.  They are consecutive in TILE scan
                                 // (6.5.1): raster order inside the CTB columns [tile_x0, tile_x1) -- the whole picture width without tiles
  uint16_t tile_x0, tile_x1;
  uint32_t slice_addr_rs;        // first CTB of the slice (not segment) this sub-stream belongs to
  int32_t slice_idx;             // region (SliceInfo) index: slice x tile
  int32_t slice_qp;
  uint8_t sao_luma, sao_chroma;
  uint8_t init_contexts;         // 1: first sub-stream of an independent slice segment
  uint8_t last_of_segment;       // 1: end_of_slice_segment_flag must be 1 at ctb_end - 1
  int32_t prev;                  // sub-stream whose end state this one continues (dependent slice segment), else -1
  // Ready-queue scheduling of the device front-end (filled by the decoder object, batch-wide sub-stream indices, -1 = none):
  int32_t wake_ctb2;             // sub-stream that becomes startable once this one has stored the contexts after its 2nd CTB of a row (9.3.2.2)
  int32_t wake_end;              // sub-stream that continues this one's end state (dependent slice segment)
  uint32_t deps;                 // number of such events this sub-stream waits for before it may start
};

struct PicBuffers {              // per-picture arrays (host memory on the host path, HBM on the device path)
  const uint8_t* rbsp; uint32_t rbsp_size;   // padded with >= 8 zero bytes
  TuCmd* tus; CoefEntry* coefs; CtuInfo* ctus; const SliceInfo* slices;
  const uint16_t* ctu_slice;     // slice index of every CTB, filled by the host from the slice headers BEFORE decoding (read-only)
  int8_t* qp8; uint8_t* edge8;   // outputs for deblocking (and QP prediction)
  uint8_t* ipm4;                 // luma intra mode per 4x4 (MPM derivation)
  uint8_t* cd8;                  // coding quadtree depth per 8x8 (split_cu_flag context)
  uint8_t* wpp_ctx;              // hctb x CTX_STRIDE: context state after the 2nd CTB of each row
  uint8_t* end_state;            // per sub-stream x CTX_STRIDE: contexts (+ last QpY in byte CTX_COUNT) at its end
};

// ---------------------------------------------------------------------------------------------- CABAC (9.3.4.3)
// Arithmetic decoder in the "scaled window" form: `val` holds the specification's 9-bit ivlOffset in bits 31..16 (as
// offset << 16) followed by up to 16 look-ahead bits; DecodeDecision / DecodeBypass / DecodeTerminate become a few
// branch-free integer operations and two table look-ups (rangeTabLps packed per state, merged state-transition table).
// The bit position after a terminating bin is reconstructed exactly (bits consumed = 9 + renormalisation shifts), which
// the host front-end cross-checks against the entry points of every WPP stream it parses.
B200_TABLE(uint8_t, kNextState, [256], {2,3,4,5,6,7,8,9,10,11,12,13,14,15,16,17,18,19,20,21,22,23,24,25,26,27,28,29,30,31,32,33,34,35,36,37,38,39,40,41,42,43,44,45,46,47,48,49,50,51,52,53,54,55,56,57,58,59,60,61,62,63,64,65,66,67,68,69,70,71,72,73,74,75,76,77,78,79,80,81,82,83,84,85,86,87,88,89,90,91,92,93,94,95,96,97,98,99,100,101,102,103,104,105,106,107,108,109,110,111,112,113,114,115,116,117,118,119,120,121,122,123,124,125,124,125,126,127,1,0,0,1,2,3,4,5,4,5,8,9,8,9,10,11,12,13,14,15,16,17,18,19,18,19,22,23,22,23,24,25,26,27,26,27,30,31,30,31,32,33,32,33,36,37,36,37,38,39,38,39,42,43,42,43,44,45,44,45,46,47,48,49,48,49,50,51,52,53,52,53,54,55,54,55,56,57,58,59,58,59,60,61,60,61,60,61,62,63,64,65,64,65,66,67,66,67,66,67,68,69,68,69,70,71,70,71,70,71,72,73,72,73,72,73,74,75,74,75,74,75,76,77,76,77,126,127})   // [ctx byte | lps << 7] -> next ctx byte ((pStateIdx << 1) | valMps)

// Both tables fused, one 64-bit entry per context byte (pStateIdx << 1 | valMps): bits 0-31 rangeTabLps[0..3], 32-39 next
// context byte after an MPS, 40-47 after an LPS, 56-62 the context byte itself.  A context variable HOLDS its entry (8 bytes),
// so a bin costs one shared-memory load on the dependency chain; the entry of the next state is fetched off the chain.
B200_TABLE(uint64_t, kState, [128], {0x00000102f0d0b080ull,0x01000003f0d0b080ull,0x02000004e3c5a780ull,0x03000105e3c5a780ull,0x04000206d8bb9e80ull,0x05000307d8bb9e80ull,0x06000408cdb2967bull,0x07000509cdb2967bull,0x0800040ac3a98e74ull,0x0900050bc3a98e74ull,0x0a00080cb9a0876full,0x0b00090db9a0876full,0x0c00080eaf988069ull,0x0d00090faf988069ull,0x0e000a10a6907a64ull,0x0f000b11a6907a64ull,0x10000c129e89745full,0x11000d139e89745full,0x12000e1496826e5aull,0x13000f1596826e5aull,0x140010168e7b6855ull,0x150011178e7b6855ull,0x1600121887756351ull,0x1700131987756351ull,0x1800121a806f5e4dull,0x1900131b806f5e4dull,0x1a00161c7a695949ull,0x1b00171d7a695949ull,0x1c00161e74645545ull,0x1d00171f74645545ull,0x1e0018206e5f5042ull,0x1f0019216e5f5042ull,0x20001a22685a4c3eull,0x21001b23685a4c3eull,0x22001a246356483bull,0x23001b256356483bull,0x24001e265e514538ull,0x25001f275e514538ull,0x26001e28594d4135ull,0x27001f29594d4135ull,0x2800202a55493e33ull,0x2900212b55493e33ull,0x2a00202c50453b30ull,0x2b00212d50453b30ull,0x2c00242e4c42382eull,0x2d00252f4c42382eull,0x2e002430483f352bull,0x2f002531483f352bull,0x30002632453b3229ull,0x31002733453b3229ull,0x3200263441383027ull,0x3300273541383027ull,0x34002a363e362d25ull,0x35002b373e362d25ull,0x36002a383b332b23ull,0x37002b393b332b23ull,0x38002c3a38302921ull,0x39002d3b38302921ull,0x3a002c3c352e2720ull,0x3b002d3d352e2720ull,0x3c002e3e322b251eull,0x3d002f3f322b251eull,0x3e0030403029231dull,0x3f0031413029231dull,0x400030422d27211bull,0x410031432d27211bull,0x420032442b251f1aull,0x430033452b251f1aull,0x4400344629231e18ull,0x4500354729231e18ull,0x4600344827211c17ull,0x4700354927211c17ull,0x4800364a25201b16ull,0x4900374b25201b16ull,0x4a00364c231e1a15ull,0x4b00374d231e1a15ull,0x4c00384e211d1814ull,0x4d00394f211d1814ull,0x4e003a501f1b1713ull,0x4f003b511f1b1713ull,0x50003a521e1a1612ull,0x51003b531e1a1612ull,0x52003c541c191511ull,0x53003d551c191511ull,0x54003c561b171410ull,0x55003d571b171410ull,0x56003c581916130full,0x57003d591916130full,0x58003e5a1815120eull,0x59003f5b1815120eull,0x5a00405c1714110eull,0x5b00415d1714110eull,0x5c00405e1613100dull,0x5d00415f1613100dull,0x5e00426015120f0cull,0x5f00436115120f0cull,0x6000426214110e0cull,0x6100436314110e0cull,0x6200426413100e0bull,0x6300436513100e0bull,0x64004466120f0d0bull,0x65004567120f0d0bull,0x66004468110f0c0aull,0x67004569110f0c0aull,0x6800466a100e0c0aull,0x6900476b100e0c0aull,0x6a00466c0f0d0b09ull,0x6b00476d0f0d0b09ull,0x6c00466e0e0c0b09ull,0x6d00476f0e0c0b09ull,0x6e0048700e0c0a08ull,0x6f0049710e0c0a08ull,0x700048720d0b0908ull,0x710049730d0b0908ull,0x720048740c0b0907ull,0x730049750c0b0907ull,0x74004a760c0a0907ull,0x75004b770c0a0907ull,0x76004a780b0a0807ull,0x77004b790b0a0807ull,0x78004a7a0b090806ull,0x79004b7b0b090806ull,0x7a004c7c0a090706ull,0x7b004d7d0a090706ull,0x7c004c7c09080706ull,0x7d004d7d09080706ull,0x7e007e7e02020202ull,0x7f007f7f02020202ull})

// The sub-stream's bytes (cold: touched once per 16 consumed bits).
struct CabacStream { const uint8_t* d; uint32_t size; };

// Arithmetic decoder (9.3.4.3) in scaled-window form: val = offset << 16 | look-ahead bits; five scalars that stay in
// registers inside the residual decoder.  The stream is consumed 16 bits at a time and the next 16 bits are always
// already loaded (next16), so the load latency never sits on the bin-to-bin dependency chain.
struct Cabac {
  uint32_t val, range; int bits;                      // bits: valid look-ahead bits in the low half of val
  uint32_t pos, next16;                               // byte offset of the 16 bits that follow next16's
  TabPtr state_tab;                                   // kState (its shared-window address is not free to form on the device)
  // big-endian 16 bits at EVEN byte offset p; offsets past the end read the zero padding the buffer ends in (>= 2 bytes, size even)
  B200_HD static inline uint32_t fetch16(const CabacStream& st, uint32_t p) {
    const uint32_t q = p < st.size - 2 ? p : st.size - 2;
#ifdef B200_SYN_DEVICE
    return __byte_perm((uint32_t)__ldg(reinterpret_cast<const unsigned short*>(st.d + q)), 0, 0x4401);
#else
    return ((uint32_t)st.d[q] << 8) | st.d[q + 1];
#endif
  }
#ifdef B200_SYN_DEVICE
  // out of line ON PURPOSE: a call inside the refill keeps ptxas from if-converting (predicating) its ~10 instructions into
  // every bin -- they are needed once per 16 consumed bits
  static __device__ __noinline__ uint32_t fetch16_cold(const uint8_t* d, uint32_t q) { return __byte_perm((uint32_t)__ldg(reinterpret_cast<const unsigned short*>(d + q)), 0, 0x4401); }
#else
  static inline uint32_t fetch16_cold(const uint8_t* d, uint32_t q) { return ((uint32_t)d[q] << 8) | d[q + 1]; }
#endif
  B200_HD inline void start(const CabacStream& st, uint32_t start_byte) {
    // initial window: the 9 bits of 9.3.2.5 + look-ahead up to the next even byte offset (2 or 3 bytes), so that every
    // later refill is one aligned 16-bit load
    if (start_byte & 1) {
      const uint32_t b0 = fetch16(st, start_byte - 1) & 0xffu, w1 = fetch16(st, start_byte + 1);
      val = ((b0 << 16) | w1) << 1; bits = 15; pos = start_byte + 3;
    } else {
      val = fetch16(st, start_byte) << 9; bits = 7; pos = start_byte + 2;
    }
    range = 510; next16 = fetch16(st, pos);
    state_tab = B200_TADDR(kState);
  }
  B200_HD inline uint64_t bit_position() const { return (uint64_t)pos * 8 - (uint32_t)bits; }
  // shift the window left by n (n <= 7), merging the prefetched 16 bits when the look-ahead is exhausted
  // (inline: a call here costs a convergence barrier and argument set-up at every one of the ~15 sites it is inlined into)
  B200_HD inline void shift(int n, const CabacStream& st) {
    val <<= n; bits -= n;
    if (bits < 0) { val |= next16 << (-bits); bits += 16; pos += 2; next16 = fetch16_cold(st.d, pos < st.size - 2 ? pos : st.size - 2); }
  }
  // One context-coded bin with the context's entry `e` already in registers; `ne` returns the entry written back (the
  // caller forwards it when the next bin uses the same context and was fetched before this store).
  B200_HD inline int bin_e(const U2 e, CtxPtr c, const CabacStream& st, U2& ne) {
#ifdef B200_SYN_DEVICE
    uint32_t rlps; asm("prmt.b32 %0, 0, %1, %2;" : "=r"(rlps) : "r"(e.x), "r"(range >> 6));   // range in [256, 510]: selector 4..7 = byte (range >> 6) & 3 of e.x
#else
    const uint32_t rlps = (e.x >> (((range >> 6) & 3) * 8)) & 0xff;
#endif
    const uint32_t rmps = range - rlps, t = rmps << 16;
    const bool lps = val >= t;
    if (lps) val -= t;
    range = lps ? rlps : rmps;
    ne = tab_ld64(state_tab, (int)((lps ? e.y >> 8 : e.y) & 0xffu));
    ctx_st(c, ne);
#ifdef B200_SYN_DEVICE
    const int n = __clz((int)range) - 23;
#else
    const int n = __builtin_clz(range) - 23;
#endif
    range <<= n;
    shift(n, st);
    return (int)(((e.y >> 24) ^ (lps ? 1u : 0u)) & 1u);
  }
  B200_HD inline int bin(CtxPtr c, const CabacStream& st) { U2 ne; return bin_e(ctx_ld(c), c, st, ne); }
  B200_HD inline int bypass(const CabacStream& st) {
    shift(1, st);
    const uint32_t one = (val >> 16) >= range ? 1u : 0u;
    val -= one ? (range << 16) : 0u;
    return (int)one;
  }
  // k bypass bins at once (9.3.4.3.4 applied k times): offset < range, so (offset << k | bits) / range < 2^k is the bin string
  B200_HD inline unsigned bypass_bits(int k, const CabacStream& st) {
    unsigned out = 0;
    B200_NOUNROLL while (k > 0) {
      const int t = k > 7 ? 7 : k;                       // window (9 bits) + t <= 16 bits: stays inside bits 31..16 of val
      shift(t, st);
      const uint32_t w = val >> 16;                      // (offset << t) | t fresh bits, < 2^16
#ifdef B200_SYN_DEVICE
      uint32_t q = (uint32_t)__float2int_rz(__fdividef((float)w, (float)range));   // within 1 of the quotient; fixed up exactly below
      int r = (int)w - (int)(q * range);
      if (r < 0) { q--; r += (int)range; } else if (r >= (int)range) { q++; r -= (int)range; }
      val = ((uint32_t)r << 16) | (val & 0xffffu);
#else
      const uint32_t q = w / range;
      val -= (q * range) << 16;
#endif
      out = (out << t) | (q & ((1u << t) - 1u)); k -= t;       // (the mask only matters for corrupt data: an offset >= range, 9.3.2.5)
    }
    return out;
  }
  B200_HD inline int terminate(const CabacStream& st) {
    range -= 2;
    if ((val >> 16) >= range) return 1;
    if (range < 256) { range <<= 1; shift(1, st); }
    return 0;
  }
};

B200_HDN inline void init_contexts(CtxPtr ctx, int slice_qp) {          // 9.3.2.2
  const int qp = clip3(0, 51, slice_qp);
  B200_LANES_BEGIN();
  B200_LANE_FOR(i, CTX_COUNT) {
    const int iv = B200_T(kInitI)[i], m = (iv >> 4) * 5 - 45, nn = ((iv & 15) << 3) - 16;
    const int pre = clip3(1, 126, ((m * qp) >> 4) + nn);
    const int mps = pre > 63, st = mps ? pre - 64 : 63 - pre;
    ctx_st(ctx_at(ctx, i), tab_ld64(B200_TADDR(kState), (st << 1) | mps));
  }
  B200_LANES_END();
}

// context states from the bytes (pStateIdx << 1 | valMps) another sub-stream stored (WPP hand-over, dependent segment)
B200_HDN inline void load_contexts(CtxPtr ctx, const uint8_t* st) {
  B200_LANES_BEGIN();
  B200_LANE_FOR(i, CTX_COUNT) ctx_st(ctx_at(ctx, i), tab_ld64(B200_TADDR(kState), (int)B200_LD_SHARED(st + i) & 127));
  B200_LANES_END();
}
B200_HDN inline void store_contexts(CtxPtr ctx, uint8_t* st) {
  B200_LANES_BEGIN();
  B200_LANE_FOR(i, CTX_COUNT) st[i] = (uint8_t)(ctx_ld(ctx_at(ctx, i)).y >> 24);
  B200_LANES_END();
}

enum { SYN_OK = 0, SYN_E_BITSTREAM = 1, SYN_E_OVERFLOW = 2 };

struct SaoRaw { int8_t type[3], band[3], eo[3]; int8_t off[3][4]; };

// ---------------------------------------------------------------------------------------------- sub-stream decoder
// Compile-time stream profile: a value >= 0 replaces the SeqParams field of the same name by a constant.  The device
// front-end instantiates the decoder twice: CfgRuntime (anything the parser accepts) and CfgCommon, the parameter
// combination of x265-produced HEIC files (and of libheif/examples/example.heic: 4:2:0 8 bit, min CB 8, TB 4..32, no
// transform skip, cu_qp_delta + sign data hiding + SAO on, WPP); the kernel's speed is set by its instruction-cache
// footprint, and the constants remove ~5 KB of it.  The host front-end uses CfgRuntime.
struct CfgRuntime { enum : int { chroma = -1, bd = -1, log2_min_cb = -1, log2_min_tb = -1, log2_max_tb = -1, transform_skip = -1, cu_qp_delta = -1, sign_hiding = -1, sao_enabled = -1, wpp = -1, dense = -1, pcm = -1, tq_bypass = -1, tiles = -1 }; };
struct CfgCommon { enum : int { chroma = 1, bd = 8, log2_min_cb = 3, log2_min_tb = 2, log2_max_tb = 5, transform_skip = 0, cu_qp_delta = 1, sign_hiding = 1, sao_enabled = 1, wpp = 1, dense = 0, pcm = 0, tq_bypass = 0, tiles = 0 }; };
B200_HD inline bool matches_common(const SeqParams& q) {
  return q.chroma == 1 && q.bd == 8 && q.log2_min_cb == 3 && q.log2_min_tb == 2 && q.log2_max_tb == 5 && !q.transform_skip && q.cu_qp_delta == 1 && q.sign_hiding == 1 &&
         q.sao_enabled == 1 && q.wpp == 1 && q.dense == 0 && !q.pcm && !q.tq_bypass && !q.tiles;
}
#define B200_SPC(f) ((int)Cfg::f >= 0 ? (int)Cfg::f : (int)sp->f)
#define B200_SPR(f) ((int)Cfg::f >= 0 ? (int)Cfg::f : (int)sp.f)

template <class Cfg>
struct DecoderT {
  const SeqParams* sp; PicBuffers pb; const Substream* ss;
  Cabac cabac; CabacStream stream; CtxPtr ctx;    // ctx: CTX_COUNT context states (caller-provided storage)
  int is_dqp_coded, dqp_val, qpy_prev_qg, last_cu_qpy, first_qg, cur_qpy, err;
  int cu_bypass;                                  // cu_transquant_bypass_flag of the current coding unit
  uint32_t tu_n, coef_n, tu_cap, coef_cap;        // write cursors / limits of the current CTB (or of the picture when dense)
  uint32_t ctb_tu0;                               // first TU of the current CTB
  int cur_ctb_x, cur_ctb_y;
  int ctb_x0, ctb_y0, left_ok, up_ok;            // current CTB: origin, availability of the CTB to the left / above (same region: slice and tile)
  int left_lf, up_lf;                            // deblocking across the CTB's left / upper boundary is allowed (8.7.2.3: slice and tile rules)
  struct Cu { int x0, y0, log2cb, nxn, lmode[4], cmode; int cmodes[4]; };   // cmodes: IntraPredModeC per prediction unit (4:4:4: one per PU; 4:2:2: [0], after Table 8-3)

  // 6.4.1 for the LEFT (x - 1, y) or ABOVE (x, y - 1) neighbour of a position inside the current CTB -- the only queries
  // the intra syntax makes.  Such a neighbour precedes the block in decoding order, so it is available iff it lies in the
  // picture and in the same slice (HEVC tiles are not supported): always inside the current CTB, else decided once per CTB.
  B200_HD inline bool avail(int x, int y) const { return x >= ctb_x0 ? (y >= ctb_y0 ? true : up_ok != 0) : left_ok != 0; }
  // Map cells of this CTB row were written by this very thread (plain load, L1); cells of the row above by another
  // sub-stream's thread, possibly on another SM (L1-bypassing load).
  B200_HD inline int ld_cell(const uint8_t* p, int y) const { return y >= ctb_y0 ? (int)*p : (int)B200_LD_SHARED(p); }

  // Out-of-line arithmetic-decoder primitives for everything outside residual_coding (which keeps its own register
  // copy of the decoder): a call instead of ~35 inlined instructions per syntax element keeps the hot code small.
  B200_HDN int dbin(int ci) { return cabac.bin(ctx_at(ctx, ci), stream); }
  B200_HDN int dbypass() { return cabac.bypass(stream); }
  B200_HDN unsigned dbits(int k) { return cabac.bypass_bits(k, stream); }

  // -------- SAO (7.3.8.3)
  B200_HDN void parse_sao(int rx, int ry, CtuInfo& ci) {
    const int addr = ry * sp->wctb + rx;
    B200_NOUNROLL for (int c = 0; c < 3; c++) { ci.sao[c].type = 0; ci.sao[c].band_or_class = 0; B200_NOUNROLL for (int k = 0; k < 4; k++) ci.sao[c].offset[k] = 0; }
    if (!ss->sao_luma && !ss->sao_chroma) return;
    int ml = 0, mu = 0;
    if (left_ok) ml = dbin(CTX_SAO_MERGE);                        // leftCtbInSliceSeg && leftCtbInTile (7.3.8.3)
    if (up_ok && !ml) mu = dbin(CTX_SAO_MERGE);
    if (ml || mu) {
      const unsigned long long* o = reinterpret_cast<const unsigned long long*>(pb.ctus[ml ? addr - 1 : addr - sp->wctb].sao);   // 3 x 8 bytes
      unsigned long long* dsto = reinterpret_cast<unsigned long long*>(ci.sao);
      B200_NOUNROLL for (int c = 0; c < 3; c++) dsto[c] = B200_LD_SHARED(o + c);
      return;
    }
    B200_NOUNROLL for (int c = 0; c < (B200_SPC(chroma) ? 3 : 1); c++) {
      if ((c == 0 && !ss->sao_luma) || (c > 0 && !ss->sao_chroma)) continue;
      if (c < 2) { int t = 0; if (dbin(CTX_SAO_TYPE)) t = dbypass() ? 2 : 1; ci.sao[c].type = (uint8_t)t; } else ci.sao[2].type = ci.sao[1].type;
      if (!ci.sao[c].type) continue;
      const int cmax = (1 << (imin(B200_SPC(bd), 10) - 5)) - 1;
      int av[4];
      B200_NOUNROLL for (int i = 0; i < 4; i++) { int v = 0; B200_NOUNROLL while (v < cmax && dbypass()) v++; av[i] = v; }
      const int sc = c == 0 ? sp->sao_scale_luma : sp->sao_scale_chroma;
      if (ci.sao[c].type == 1) {
        B200_NOUNROLL for (int i = 0; i < 4; i++) if (av[i] && dbypass()) av[i] = -av[i];
        ci.sao[c].band_or_class = (uint8_t)dbits(5);
        B200_NOUNROLL for (int i = 0; i < 4; i++) ci.sao[c].offset[i] = (int8_t)clip3(-128, 127, av[i] * (1 << sc));
      } else {
        if (c < 2) ci.sao[c].band_or_class = (uint8_t)dbits(2); else ci.sao[2].band_or_class = ci.sao[1].band_or_class;
        ci.sao[c].offset[0] = (int8_t)clip3(-128, 127, av[0] << sc); ci.sao[c].offset[1] = (int8_t)clip3(-128, 127, av[1] << sc);
        ci.sao[c].offset[2] = (int8_t)clip3(-128, 127, -(av[2] << sc)); ci.sao[c].offset[3] = (int8_t)clip3(-128, 127, -(av[3] << sc));
      }
    }
  }

  // -------- QP (8.6.1); QpY is kept per 8x8 block (coding blocks are >= 8x8)
  B200_HDN void derive_qpy(int xcb, int ycb) {
    const int mask = (1 << sp->qg_log2) - 1, xqg = xcb & ~mask, yqg = ycb & ~mask, cm = ~((1 << sp->log2ctb) - 1);
    int qa = qpy_prev_qg, qb = qpy_prev_qg;
    if (avail(xqg - 1, yqg) && ((xqg - 1) & cm) == (xqg & cm)) qa = pb.qp8[(yqg >> 3) * sp->w8 + ((xqg - 1) >> 3)];   // same CTB: own data
    if (avail(xqg, yqg - 1) && ((yqg - 1) & cm) == (yqg & cm)) qb = pb.qp8[((yqg - 1) >> 3) * sp->w8 + (xqg >> 3)];
    const int pred = (qa + qb + 1) >> 1, qbd = 6 * (B200_SPC(bd) - 8);
    cur_qpy = ((pred + dqp_val + 52 + 2 * qbd) % (52 + qbd)) - qbd;
  }

  // -------- residual_coding (7.3.8.11): emits sparse (pos, level) entries; returns the number of coefficients
  B200_HDN int residual(int log2n, int c, int mode, int& tskip) {
    const int n = 1 << log2n;
    // Local copies: their addresses never escape, so they live in registers.
    Cabac cb_ = cabac; const CtxPtr cx = ctx;
    const int bypass_cu = B200_SPC(tq_bypass) && cu_bypass;            // 7.3.8.11: no transform_skip_flag, no sign data hiding
    const int sign_hiding = B200_SPC(sign_hiding) && !bypass_cu;
    uint32_t cn = coef_n;
    tskip = 0;
    if (B200_SPC(transform_skip) && log2n == 2 && !bypass_cu) tskip = cb_.bin(ctx_at(cx, CTX_TSKIP + (c ? 1 : 0)), stream);
    const int cmax = (log2n << 1) - 1;
    int off, shift;
    if (c == 0) { off = 3 * (log2n - 2) + ((log2n - 1) >> 2); shift = (log2n + 1) >> 2; } else { off = 15; shift = log2n - 2; }
    int lx = 0, ly = 0;
    // last_sig_coeff_{x,y}_prefix then the two suffixes (7.3.8.11 order); one loop body serves both coordinates.  The entry
    // of the context the NEXT bin would use is fetched before the current bin is decoded (it is needed only if that bin is
    // 1); when it is the same context, the freshly written entry is forwarded in registers.
    B200_NOUNROLL for (int xy = 0; xy < 2; xy++) {
      const CtxPtr lc = ctx_at(cx, (xy ? CTX_LAST_Y : CTX_LAST_X) + off);
      int l = 0;
      CtxPtr a_cur = lc; U2 e_cur = ctx_ld(a_cur);
      B200_NOUNROLL while (l < cmax) {
        const CtxPtr a_next = ctx_at(lc, (l + 1) >> shift);
        U2 e_next = ctx_ld(a_next), ne;
        const int b = cb_.bin_e(e_cur, a_cur, stream, ne);
        if (!b) break;
        if (a_next == a_cur) e_next = ne;
        a_cur = a_next; e_cur = e_next; l++;
      }
      if (xy) ly = l; else lx = l;
    }
    B200_NOUNROLL for (int xy = 0; xy < 2; xy++) {
      int l = xy ? ly : lx;
      if (l > 3) { const int nb = (l >> 1) - 1; l = (1 << nb) * (2 + (l & 1)) + (int)cb_.bypass_bits(nb, stream); }
      if (xy) ly = l; else lx = l;
    }
    int scan = 0;
    if (log2n == 2 || (log2n == 3 && (c == 0 || B200_SPC(chroma) == 3))) { if (mode >= 6 && mode <= 14) scan = 2; else if (mode >= 22 && mode <= 30) scan = 1; }
    if (scan == 2) { const int t = lx; lx = ly; ly = t; }
    if (lx >= n || ly >= n) { err = SYN_E_BITSTREAM; cabac = cb_; return 0; }
    const int l2sb = log2n - 2;
    const TabPtr sbx = B200_TADDR(kScanX) + 64 * (3 * l2sb + scan), sby = B200_TADDR(kScanY) + 64 * (3 * l2sb + scan), spos = B200_TADDR(kScanPos) + 16 * scan;
    const int last_sb = B200_T(kSbInv)[l2sb][scan][((ly >> 2) << 3) + (lx >> 2)];
    const int last_pos = B200_T(kScanInv)[scan][((ly & 3) << 2) + (lx & 3)];
    uint64_t csbf = 0;                                  // coded_sub_block_flag, bit (ys * 8 + xs)
    int carry = 1;                                      // greater1Ctx carried over (9.3.4.2.6); not 0 before the first coded sub-block
    const int sig_base = log2n == 2 ? CTX_SIG + (c ? 27 : 0) : (c == 0 ? CTX_SIG + (log2n == 3 ? (scan == 0 ? 9 : 15) : 21) : CTX_SIG + 27 + (log2n == 3 ? 9 : 12));
    B200_NOUNROLL for (int i = last_sb; i >= 0; i--) {
      const int xs = (int)tab_ld8(sbx, i), ys = (int)tab_ld8(sby, i);
      const int right = ((xs + 1) >> l2sb) == 0 ? (int)((csbf >> (ys * 8 + xs + 1)) & 1) : 0;
      const int below = ((ys + 1) >> l2sb) == 0 ? (int)((csbf >> ((ys + 1) * 8 + xs)) & 1) : 0;
      const bool is_last = csbf == 0;                   // the sub-block of the last significant coefficient is the first one coded
      int infer_dc = 0;
      if (!is_last && i > 0) { if (!cb_.bin(ctx_at(cx, CTX_CSBF + ((right | below) ? 1 : 0) + (c ? 2 : 0)), stream)) continue; infer_dc = 1; }
      csbf |= 1ull << (ys * 8 + xs);
      // sig_coeff_flag (9.3.4.2.5): context = per-sub-block base + table entry per scan position; DC of the block has its own
      const TabPtr tab = log2n == 2 ? B200_TADDR(kSigCtx4) + 16 * scan : B200_TADDR(kSigCtxN) + (64 * scan + 16 * (right | (below << 1)));
      const CtxPtr cbase = ctx_at(cx, sig_base + ((c == 0 && log2n > 2 && (xs | ys)) ? 3 : 0));
      // flags are shifted in from the right: after the last position (k = 0) bit k of `sig` is the flag of scan position k
      unsigned sig = 0;
      int k = 15;
      if (is_last) { sig = 1u; k = last_pos - 1; }
      if (k >= 0) {
        // software pipeline: the entry of position k - 1 is in flight while position k is decoded (the contexts depend on the
        // position only, 9.3.4.2.5); same context twice in a row -> forward the new entry in registers
        const CtxPtr a0 = i == 0 ? ctx_at(cx, CTX_SIG + (c ? 27 : 0)) : ctx_at(cbase, (int)tab_ld8(tab, 0));
        CtxPtr a_cur = k > 0 ? ctx_at(cbase, (int)tab_ld8(tab, k)) : a0;
        U2 e_cur = ctx_ld(a_cur);
        B200_NOUNROLL for (; k > 0; k--) {
          const CtxPtr a_next = k > 1 ? ctx_at(cbase, (int)tab_ld8(tab, k - 1)) : a0;
          U2 e_next = ctx_ld(a_next), ne;
          sig = (sig << 1) | (unsigned)cb_.bin_e(e_cur, a_cur, stream, ne);
          if (a_next == a_cur) e_next = ne;
          a_cur = a_next; e_cur = e_next;
        }
        if (infer_dc && !sig) sig = 1u;
        else { U2 ne; sig = (sig << 1) | (unsigned)cb_.bin_e(e_cur, a_cur, stream, ne); }
      }
      if (!sig) continue;
      unsigned g1 = 0;
      int g1ctx = 1, g2 = 0;
      int ctx_set = (i == 0 || c > 0) ? 0 : 2;
      if (carry == 0) ctx_set++;
      const int last_sig = hi_bit(sig), first_sig = lo_bit(sig);
      { unsigned m = sig; const CtxPtr gbase = ctx_at(cx, CTX_GT1 + ctx_set * 4 + (c ? 16 : 0));
        B200_NOUNROLL for (int ng1 = 0; m && ng1 < 8; ng1++) {
          const int kk = hi_bit(m); m ^= 1u << kk;
          if (cb_.bin(ctx_at(gbase, imin(3, g1ctx)), stream)) { g1 |= 1u << kk; g1ctx = 0; } else if (g1ctx > 0) g1ctx++;
        } }
      carry = g1ctx;
      const int last_g1 = g1 ? hi_bit(g1) : -1;           // the first coefficient (in decoding order) with a greater1 flag of 1
      const bool hidden = sign_hiding && (last_sig - first_sig > 3);
      if (last_g1 >= 0) g2 = cb_.bin(ctx_at(cx, CTX_GT2 + ctx_set + (c ? 4 : 0)), stream);
      const int nsign = pop_count(sig) - (hidden ? 1 : 0);
      const unsigned signs = cb_.bypass_bits(nsign, stream);
#ifdef B200_SYN_DEVICE
      // The serial loop keeps what is serial by nature (the coeff_abs_level_remaining bins, Rice adaptation, the parity sum
      // of sign hiding) and leaves each absolute level in the warp's scratch words behind its context array; then lane k < 16
      // emits scan position k: output index (significant positions above it), sign, position, clip, one store.
      int nsig = 0, sum = 0, rice = 0;
      const uint32_t lv = ctx_at(cx, CTX_COUNT);
      B200_NOUNROLL for (unsigned m = sig; m; nsig++) {
        const int kk = hi_bit(m); m ^= 1u << kk;
        const int base = 1 + (int)((g1 >> kk) & 1) + (kk == last_g1 ? g2 : 0);
        int a = base;
        if (base == ((nsig < 8) ? ((kk == last_g1) ? 3 : 2) : 1)) {
          int pre = 0; B200_NOUNROLL while (pre < 32 && cb_.bypass(stream)) pre++;
          if (pre > 20) { err = SYN_E_BITSTREAM; cabac = cb_; const int count = (int)(cn - coef_n); coef_n = cn; return count; }   // far outside the 16-bit range of TransCoeffLevel: corrupt data
          const int rem = (pre <= 3 ? (pre << rice) : (((1 << (pre - 3)) + 3 - 1) << rice)) + (int)cb_.bypass_bits(pre <= 3 ? rice : pre - 3 + rice, stream);
          a = base + rem;
          if (a > 3 * (1 << rice)) rice = imin(rice + 1, 4);
        }
        sum += a;
        asm volatile("st.shared.u32 [%0], %1;" ::"r"(lv + 4u * (uint32_t)kk), "r"(a));
      }
      if (cn + (uint32_t)nsig > coef_cap) { err = SYN_E_OVERFLOW; cabac = cb_; const int count = (int)(cn - coef_n); coef_n = cn; return count; }
      B200_LANES_BEGIN();
      { const int k = lane_id();
        if (k < 16 && ((sig >> k) & 1u)) {
          int a; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(a) : "r"(lv + 4u * (uint32_t)k));
          const int above = pop_count(sig >> k >> 1);     // coefficients decoded (and emitted) before this one
          const int neg = (hidden && k == first_sig) ? (sum & 1) : (int)((signs >> (nsign - 1 - above)) & 1u);
          const int p = (int)tab_ld8(spos, k);
          CoefEntry e; e.pos = (uint16_t)((((ys << 2) + (p >> 2)) << log2n) + (xs << 2) + (p & 3)); e.level = (int16_t)clip3(-32768, 32767, neg ? -a : a);
          pb.coefs[cn + (uint32_t)above] = e;
        } }
      B200_LANES_END();
      cn += (uint32_t)nsig;
#else
      int nsig = 0, sum = 0, rice = 0, sidx = nsign;
      B200_NOUNROLL for (unsigned m = sig; m; nsig++) {
        const int kk = hi_bit(m); m ^= 1u << kk;
        const int base = 1 + (int)((g1 >> kk) & 1) + (kk == last_g1 ? g2 : 0);
        int a = base;
        if (base == ((nsig < 8) ? ((kk == last_g1) ? 3 : 2) : 1)) {
          int pre = 0; B200_NOUNROLL while (pre < 32 && cb_.bypass(stream)) pre++;
          if (pre > 20) { err = SYN_E_BITSTREAM; cabac = cb_; const int count = (int)(cn - coef_n); coef_n = cn; return count; }   // far outside the 16-bit range of TransCoeffLevel: corrupt data
          const int rem = (pre <= 3 ? (pre << rice) : (((1 << (pre - 3)) + 3 - 1) << rice)) + (int)cb_.bypass_bits(pre <= 3 ? rice : pre - 3 + rice, stream);
          a = base + rem;
          if (a > 3 * (1 << rice)) rice = imin(rice + 1, 4);
        }
        int neg = 0;
        if (!hidden || kk != first_sig) { sidx--; neg = (int)((signs >> sidx) & 1); }
        int v = neg ? -a : a;
        if (hidden) { sum += a; if (kk == first_sig && (sum & 1)) v = -v; }
        if (cn >= coef_cap) { err = SYN_E_OVERFLOW; cabac = cb_; const int count = (int)(cn - coef_n); coef_n = cn; return count; }
        const int p = (int)tab_ld8(spos, kk);
        CoefEntry e; e.pos = (uint16_t)((((ys << 2) + (p >> 2)) << log2n) + (xs << 2) + (p & 3)); e.level = (int16_t)clip3(-32768, 32767, v);
        pb.coefs[cn++] = e;
      }
#endif
    }
    cabac = cb_;
    const int count = (int)(cn - coef_n);                 // coefficients written
    coef_n = cn;
    return count;
  }

  // -------- transform tree / unit (7.3.8.8, 7.3.8.10)
  B200_HDN void mark_tu(int x0, int y0, int log2n) {
    // QpY map + filterEdgeFlag (8.7.2.3, bS = 2 on every transform edge of the 8x8 grid) for the deblocking kernel
    const SliceInfo& sl = pb.slices[ss->slice_idx];
    const int n8 = log2n > 3 ? 1 << (log2n - 3) : 1, bx = x0 >> 3, by = y0 >> 3;
    uint8_t left = 0, top = 0;
    if (!sl.deblocking_disabled) {
      if ((x0 & 7) == 0 && x0 > 0 && (x0 > ctb_x0 || left_lf)) left = 1;
      if ((y0 & 7) == 0 && y0 > 0 && (y0 > ctb_y0 || up_lf)) top = 2;
    }
    // the CTB's flags were cleared in decode_ctb: only the first column / row of 8x8 cells carries an edge.  (QpY of the
    // cells is written once per coding unit, at its end.)  Item k < n8: cell k of the column (the corner takes both flags);
    // k >= n8: cell k - n8 + 1 of the row -- no two items touch the same cell.
    uint8_t* e = pb.edge8 + by * sp->w8 + bx;
    if (!(left | top)) return;
    B200_LANES_BEGIN();
    B200_LANE_FOR(k, 2 * n8 - 1) {
      const bool col = k < n8;
      const uint8_t v = col ? (uint8_t)(left | (k ? 0 : top)) : top;
      if (v) e[col ? k * sp->w8 : k - n8 + 1] |= v;
    }
    B200_LANES_END();
  }

  B200_HDI void transform_unit(const Cu& cu, int x0, int y0, int log2n, int blk, int cbf_l, int cbf_cb, int cbf_cr, int pcb, int pcr) {
    const int cbf_c = B200_SPC(chroma) ? (log2n > 2 ? (cbf_cb | cbf_cr) : (pcb | pcr)) : 0;
    if ((cbf_l || cbf_c) && B200_SPC(cu_qp_delta) && !is_dqp_coded) {
      int v = 0;
      B200_NOUNROLL while (v < 5 && dbin(CTX_QP_DELTA + (v ? 1 : 0))) v++;
      if (v == 5) { int k = 0; B200_NOUNROLL while (k < 16 && dbypass()) { v += 1 << k; k++; } v += (int)dbits(k); }
      if (v && dbypass()) v = -v;
      { const int half = 3 * (B200_SPC(bd) - 8); if (v < -(26 + half) || v > 25 + half) { err = SYN_E_BITSTREAM; return; } }   // CuQpDeltaVal range (7.4.9.10)
      is_dqp_coded = 1; dqp_val = v;
      derive_qpy(cu.x0, cu.y0);
    }
    const int pu = cu.nxn ? ((y0 >= cu.y0 + (1 << (cu.log2cb - 1))) ? 2 : 0) + ((x0 >= cu.x0 + (1 << (cu.log2cb - 1))) ? 1 : 0) : 0;
    const int lmode = cu.lmode[pu];
    const uint32_t coef0 = coef_n;
    int chroma_here = 0, ccb = 0, ccr = 0;
    if (B200_SPC(chroma)) {
      if (log2n > 2) { chroma_here = 1; ccb = cbf_cb; ccr = cbf_cr; }
      else if (blk == 3) { chroma_here = 1; ccb = pcb; ccr = pcr; }      // 4x4 chroma blocks of the parent 8x8 node
    }
    // The command is assembled before the residuals and only its packed words (plus the loop counter) are live across the
    // residual_coding calls: position, size, cbf flags, modes, later the transform-skip flags and coefficient counts.
    TuCmd t;
    t.w0 = (uint32_t)(x0 >> 2) | ((uint32_t)(y0 >> 2) << 12) | ((uint32_t)(log2n - 2) << 24) | ((uint32_t)cbf_l << 26) | ((uint32_t)ccb << 27) |
           ((uint32_t)ccr << 28) | ((uint32_t)chroma_here << 29);
    t.w1 = (uint32_t)lmode | ((uint32_t)cu.cmode << 6) | ((B200_SPC(tq_bypass) && cu_bypass) ? 1u << 22 : 0u);
    t.w2 = coef0;
    t.w3 = 0;
    // one residual_coding site serves the three components (it is inlined: call frames of a lone lane cost a 128-byte
    // line of L1 per saved register)
    B200_NOUNROLL for (int c = 0; c < 3; c++) {
      if (!((t.w0 >> (26 + c)) & 1u)) continue;                          // cbf of the component
      const int l2 = (int)((t.w0 >> 24) & 3u) + 2;
      int ts = 0;
      const int cnt = residual(c == 0 ? l2 : (l2 > 2 ? l2 - 1 : 2), c, (int)((t.w1 >> (c == 0 ? 0 : 6)) & 63u), ts);
      t.w3 |= (uint32_t)cnt << (c == 0 ? 0 : (c == 1 ? 11 : 21));
      if (c == 0) t.w0 |= (uint32_t)ts << 30; else if (c == 1) t.w0 |= (uint32_t)ts << 31; else t.w1 |= (uint32_t)ts << 20;
    }
    mark_tu((int)(t.w0 & 0xfffu) << 2, (int)((t.w0 >> 12) & 0xfffu) << 2, (int)((t.w0 >> 24) & 3u) + 2);
    if (tu_n >= tu_cap) { err = SYN_E_OVERFLOW; return; }
    t.w1 |= (uint32_t)(cur_qpy + 64) << 12;
    pb.tus[tu_n++] = t;
  }

  // z-order index -> (x, y): even bits / odd bits compacted (indices < 256)
  B200_HD static inline int zx(unsigned i) { i &= 0x55u; i = (i | (i >> 1)) & 0x33u; i = (i | (i >> 2)) & 0x0fu; return (int)i; }
  // depth of the largest quadtree node that STARTS at z-order unit i (levels = depth of a single unit)
  B200_HD static inline int node_depth(unsigned i, int levels) { const int up = i ? lo_bit(i) >> 1 : levels; return levels - imin(up, levels); }

  // transform_tree (7.3.8.8) without recursion: the tree of one coding unit is walked in z-order over 4x4 units; a node
  // is entered at the coarsest depth aligned to the current unit, split flags descend, leaves advance.  (Recursion costs
  // a lone lane one 128-byte line of L1 per saved register and frame level; see run_substream.)
  B200_HDI void transform_tree(const Cu& cu, int max_depth) {
    const int levels = cu.log2cb - 2, total = 1 << (2 * levels);
    unsigned cbm = 0, crm = 0;                          // cbf_cb / cbf_cr of the node on the current path, bit = depth
    B200_NOUNROLL for (int j = 0; j < total && !err;) {
      int depth = node_depth((unsigned)j, levels);
      B200_NOUNROLL for (;;) {
        const int log2n = cu.log2cb - depth;
        const int x0 = cu.x0 + (zx((unsigned)j) << 2), y0 = cu.y0 + (zx((unsigned)j >> 1) << 2);
        const int blk = depth ? (j >> (2 * (levels - depth))) & 3 : 0;
        const int pcb = depth ? (int)((cbm >> (depth - 1)) & 1) : 0, pcr = depth ? (int)((crm >> (depth - 1)) & 1) : 0;
        int split;
        if (log2n <= B200_SPC(log2_max_tb) && log2n > B200_SPC(log2_min_tb) && depth < max_depth && !(cu.nxn && depth == 0)) split = dbin(CTX_SPLIT_TR + 5 - log2n);
        else split = (log2n > B200_SPC(log2_max_tb) || (cu.nxn && depth == 0)) ? 1 : 0;
        if (split && log2n <= 2) { err = SYN_E_BITSTREAM; break; }
        int cb = 0, cr = 0;
        if (B200_SPC(chroma)) {
          if (log2n > 2) {
            B200_NOUNROLL for (int k = 0; k < 2; k++) {
              int f = 0;
              if (depth == 0 || (k ? pcr : pcb)) f = dbin(CTX_CBF_CHROMA + depth);
              if (k) cr = f; else cb = f;
            }
          } else { cb = pcb; cr = pcr; }
        }
        cbm = (cbm & ~(1u << depth)) | ((unsigned)cb << depth); crm = (crm & ~(1u << depth)) | ((unsigned)cr << depth);
        if (split) { depth++; continue; }               // the first child starts at the same unit
        const int cl = dbin(CTX_CBF_LUMA + (depth == 0 ? 1 : 0));
        const bool big = log2n > 2;
        transform_unit(cu, x0, y0, log2n, blk, cl, big ? cb : 0, big ? cr : 0, big ? 0 : pcb, big ? 0 : pcr);
        j += 1 << (2 * (levels - depth));
        break;
      }
    }
  }

  // -------- 4:2:2 / 4:4:4 (chroma_format_idc 2 / 3): the same walk, with the chroma structure of 7.3.8.8 / 7.3.8.10 -- two
  // cbf_cb / cbf_cr flags per unit and two square chroma blocks one above the other in 4:2:2, chroma blocks down to 4x4 at
  // every leaf in 4:4:4.  Out of line, so that the 4:2:0 path above keeps its size.  Command stream: the luma block of a
  // unit is a TuCmd without chroma (chroma_here = 0); every chroma block is a TuCmd of its own that looks like a luma one
  // (position = its luma location, size, cbf, transform skip, mode, QpY, coefficients) with the component in w1 bits 23-24.
  B200_HD inline void emit_block(int comp, int lx, int ly, int log2n, int coded, int ts, int mode, uint32_t coef0, int nnz, uint32_t flags = 0) {
    if (tu_n >= tu_cap) { err = SYN_E_OVERFLOW; return; }
    TuCmd t;
    t.w0 = (uint32_t)(lx >> 2) | ((uint32_t)(ly >> 2) << 12) | ((uint32_t)(log2n - 2) << 24) | ((uint32_t)coded << 26) | ((uint32_t)ts << 30);
    t.w1 = (uint32_t)mode | ((uint32_t)mode << 6) | ((uint32_t)(cur_qpy + 64) << 12) | ((B200_SPC(tq_bypass) && cu_bypass) ? 1u << 22 : 0u) | ((uint32_t)comp << 23) | flags;
    t.w2 = coef0; t.w3 = (uint32_t)nnz;
    pb.tus[tu_n++] = t;
  }
  B200_HDN void transform_unit_x(const Cu& cu, int x0, int y0, int xb, int yb, int log2n, int blk, int cbf_l, unsigned fcb, unsigned fcr) {
    const int cfmt = B200_SPC(chroma), sx = cfmt == 3 ? 0 : 1;           // (SubHeightC is 1 in both formats)
    if ((cbf_l || fcb || fcr) && B200_SPC(cu_qp_delta) && !is_dqp_coded) {
      int v = 0;
      B200_NOUNROLL while (v < 5 && dbin(CTX_QP_DELTA + (v ? 1 : 0))) v++;
      if (v == 5) { int k = 0; B200_NOUNROLL while (k < 16 && dbypass()) { v += 1 << k; k++; } v += (int)dbits(k); }
      if (v && dbypass()) v = -v;
      { const int half = 3 * (B200_SPC(bd) - 8); if (v < -(26 + half) || v > 25 + half) { err = SYN_E_BITSTREAM; return; } }
      is_dqp_coded = 1; dqp_val = v;
      derive_qpy(cu.x0, cu.y0);
    }
    const int pu = cu.nxn ? ((y0 >= cu.y0 + (1 << (cu.log2cb - 1))) ? 2 : 0) + ((x0 >= cu.x0 + (1 << (cu.log2cb - 1))) ? 1 : 0) : 0;
    const int lmode = cu.lmode[pu], cmode = cu.cmodes[cfmt == 3 ? pu : 0];
    { int ts = 0; const uint32_t c0 = coef_n; const int cnt = cbf_l ? residual(log2n, 0, lmode, ts) : 0; emit_block(0, x0, y0, log2n, cbf_l, ts, lmode, c0, cnt); }
    mark_tu(x0, y0, log2n);
    int lc, cx, cy;                                                       // chroma block size; luma location of the (upper) chroma block
    if (log2n > 2 || cfmt == 3) { lc = cfmt == 3 ? log2n : log2n - 1; cx = x0; cy = y0; }
    else if (blk == 3) { lc = 2; cx = xb; cy = yb; }
    else return;
    const int nb = cfmt == 2 ? 2 : 1;
    B200_NOUNROLL for (int c = 1; c <= 2; c++) B200_NOUNROLL for (int t = 0; t < nb; t++) {
      const int coded = (int)(((c == 1 ? fcb : fcr) >> t) & 1u);
      int ts = 0; const uint32_t c0 = coef_n;
      const int cnt = coded ? residual(lc, c, cmode, ts) : 0;
      if (err) return;
      emit_block(c, cx, cy + (t << lc), lc, coded, ts, cmode, c0, cnt);   // (4:2:2: chroma rows = luma rows, so the lower block sits lc rows down in luma terms too)
    }
    (void)sx;
  }
  B200_HDN void transform_tree_x(const Cu& cu, int max_depth) {
    const int cfmt = B200_SPC(chroma);
    const int levels = cu.log2cb - 2, total = 1 << (2 * levels);
    unsigned cbm = 0, crm = 0;                          // cbf_cb / cbf_cr of the node on the current path: 2 bits per depth (bit 1: lower 4:2:2 block)
    B200_NOUNROLL for (int j = 0; j < total && !err;) {
      int depth = node_depth((unsigned)j, levels);
      B200_NOUNROLL for (;;) {
        const int log2n = cu.log2cb - depth;
        const int x0 = cu.x0 + (zx((unsigned)j) << 2), y0 = cu.y0 + (zx((unsigned)j >> 1) << 2);
        const int blk = depth ? (j >> (2 * (levels - depth))) & 3 : 0;
        const unsigned pcb = depth ? (cbm >> (2 * (depth - 1))) & 3u : 0u, pcr = depth ? (crm >> (2 * (depth - 1))) & 3u : 0u;
        int split;
        if (log2n <= B200_SPC(log2_max_tb) && log2n > B200_SPC(log2_min_tb) && depth < max_depth && !(cu.nxn && depth == 0)) split = dbin(CTX_SPLIT_TR + 5 - log2n);
        else split = (log2n > B200_SPC(log2_max_tb) || (cu.nxn && depth == 0)) ? 1 : 0;
        if (split && log2n <= 2) { err = SYN_E_BITSTREAM; break; }
        unsigned cb = 0, cr = 0;
        if (log2n > 2 || cfmt == 3) {
          const bool two = cfmt == 2 && (!split || log2n == 3);
          B200_NOUNROLL for (int k = 0; k < 2; k++) {
            unsigned f = 0;
            if (depth == 0 || ((k ? pcr : pcb) & 1u)) { f = (unsigned)dbin(CTX_CBF_CHROMA + depth); if (two) f |= (unsigned)dbin(CTX_CBF_CHROMA + depth) << 1; }
            if (k) cr = f; else cb = f;
          }
        } else { cb = pcb; cr = pcr; }                 // 4x4 luma blocks of an 8x8 node (4:2:2): the node's flags
        cbm = (cbm & ~(3u << (2 * depth))) | (cb << (2 * depth)); crm = (crm & ~(3u << (2 * depth))) | (cr << (2 * depth));
        if (split) { depth++; continue; }
        const int cl = dbin(CTX_CBF_LUMA + (depth == 0 ? 1 : 0));
        const int half = 1 << log2n;                  // parent origin of a depth > 0 node
        const int xb = x0 & ~((half << 1) - 1), yb = y0 & ~((half << 1) - 1);
        transform_unit_x(cu, x0, y0, xb, yb, log2n, blk, cl, cb, cr);
        j += 1 << (2 * (levels - depth));
        break;
      }
    }
  }

  // -------- 8.4.2
  B200_HDN int luma_mode(int x, int y, int prev, int mpm_idx, int rem) const {
    int ca = 1, cb = 1;
    if (avail(x - 1, y)) ca = pb.ipm4[(y >> 2) * sp->w4 + ((x - 1) >> 2)];               // this CTB row: own data
    if (avail(x, y - 1) && (y - 1) >= ((y >> sp->log2ctb) << sp->log2ctb)) cb = pb.ipm4[((y - 1) >> 2) * sp->w4 + (x >> 2)];
    int c0, c1, c2;
    if (ca == cb) { if (ca < 2) { c0 = 0; c1 = 1; c2 = 26; } else { c0 = ca; c1 = 2 + ((ca + 29) % 32); c2 = 2 + ((ca - 2 + 1) % 32); } }
    else { c0 = ca; c1 = cb; if (ca != 0 && cb != 0) c2 = 0; else if (ca != 1 && cb != 1) c2 = 1; else c2 = 26; }
    if (prev) return mpm_idx == 0 ? c0 : (mpm_idx == 1 ? c1 : c2);
    int t;
    if (c0 > c1) { t = c0; c0 = c1; c1 = t; }
    if (c0 > c2) { t = c0; c0 = c2; c2 = t; }
    if (c1 > c2) { t = c1; c1 = c2; c2 = t; }
    int m = rem;
    if (m >= c0) m++;
    if (m >= c1) m++;
    if (m >= c2) m++;
    return m;
  }

  // -------- pcm_sample() (7.3.8.7): the unit becomes ONE TuCmd whose "coefficients" are the samples in raster order,
  // already scaled to the picture's bit depth (8.4.4.1: recSamples = pcm_sample << (BitDepth - PcmBitDepth))
  B200_HD inline uint32_t rbsp_byte(uint32_t p) const {
#ifdef B200_SYN_DEVICE
    return (uint32_t)__ldg(stream.d + p);
#else
    return stream.d[p];
#endif
  }
  B200_HDN void pcm_unit(int x0, int y0, int log2cb, int depth) {
    const int n = 1 << log2cb, cfmt = B200_SPC(chroma), chroma = cfmt ? 1 : 0;
    const int sx = (cfmt == 1 || cfmt == 2) ? 1 : 0, sy = cfmt == 1 ? 1 : 0;
    const uint32_t nl = (uint32_t)(n * n), nc = chroma ? nl >> (sx + sy) : 0;
    uint32_t p = (uint32_t)((cabac.bit_position() + 7) >> 3);          // pcm_alignment_zero_bit
    const uint64_t nbits = (uint64_t)nl * (uint32_t)sp->pcm_bd_y + 2ull * nc * (uint32_t)sp->pcm_bd_c;     // a multiple of 8
    if ((uint64_t)p * 8 + nbits > (uint64_t)stream.size * 8) { err = SYN_E_BITSTREAM; return; }
    if (coef_n + nl + 2 * nc > coef_cap || tu_n >= tu_cap) { err = SYN_E_OVERFLOW; return; }
    const uint32_t coef0 = coef_n;
    uint32_t acc = 0; int have = 0;
    B200_NOUNROLL for (int c = 0; c < (chroma ? 3 : 1); c++) {
      const uint32_t cnt = c ? nc : nl; const int bd = c ? sp->pcm_bd_c : sp->pcm_bd_y, sh = c ? sp->pcm_shift_c : sp->pcm_shift_y;
      B200_NOUNROLL for (uint32_t k = 0; k < cnt; k++) {
        B200_NOUNROLL while (have < bd) { acc = (acc << 8) | rbsp_byte(p++); have += 8; }
        have -= bd;
        const uint32_t v = (acc >> have) & ((1u << bd) - 1u);
        acc &= (1u << have) - 1u;
        CoefEntry e; e.pos = (uint16_t)k; e.level = (int16_t)(v << sh);
        pb.coefs[coef_n++] = e;
      }
    }
    cabac.start(stream, p);                                             // 9.3.2.5: the arithmetic decoder starts over after the samples
    if (!B200_SPC(cu_qp_delta)) cur_qpy = ss->slice_qp; else derive_qpy(x0, y0);
    const int nofilt = sp->pcm_lf_disabled ? 4 : 0;
    { const int l4 = log2cb - 2;                       // INTRA_DC for its neighbours' mode derivation (8.4.2)
      B200_LANES_BEGIN();
      B200_LANE_FOR(k, 1 << (2 * l4)) pb.ipm4[((y0 >> 2) + (k >> l4)) * sp->w4 + (x0 >> 2) + (k & ((1 << l4) - 1))] = 1;
      B200_LANES_END(); }
    mark_tu(x0, y0, log2cb);
    { const int l8 = log2cb - 3;
      B200_LANES_BEGIN();
      B200_LANE_FOR(k, 1 << (2 * l8)) {
        const int i8 = ((y0 >> 3) + (k >> l8)) * sp->w8 + (x0 >> 3) + (k & ((1 << l8) - 1));
        pb.cd8[i8] = (uint8_t)depth; pb.qp8[i8] = (int8_t)cur_qpy; pb.edge8[i8] |= (uint8_t)nofilt;
      }
      B200_LANES_END(); }
    last_cu_qpy = cur_qpy;
    if (cfmt >= 2) {                                   // 4:2:2 / 4:4:4: one command per block, like transform_unit_x
      emit_block(0, x0, y0, log2cb, 1, 0, 1, coef0, (int)nl, 1u << 21);
      B200_NOUNROLL for (int c = 1; c <= 2; c++) {
        const uint32_t o = coef0 + nl + (uint32_t)(c - 1) * nc;
        if (cfmt == 3) emit_block(c, x0, y0, log2cb, 1, 0, 1, o, (int)nc, 1u << 21);
        else { emit_block(c, x0, y0, log2cb - 1, 1, 0, 1, o, (int)(nc >> 1), 1u << 21); emit_block(c, x0, y0 + (n >> 1), log2cb - 1, 1, 0, 1, o + (nc >> 1), (int)(nc >> 1), 1u << 21); }
      }
      return;
    }
    TuCmd t;
    t.w0 = (uint32_t)(x0 >> 2) | ((uint32_t)(y0 >> 2) << 12) | ((uint32_t)(log2cb - 2) << 24) | (1u << 26) | ((uint32_t)chroma << 27) | ((uint32_t)chroma << 28) | ((uint32_t)chroma << 29);
    t.w1 = 1u | (1u << 6) | ((uint32_t)(cur_qpy + 64) << 12) | (1u << 21) | ((B200_SPC(tq_bypass) && cu_bypass) ? 1u << 22 : 0u);
    t.w2 = coef0;
    t.w3 = nl | (nc << 11) | (nc << 21);
    pb.tus[tu_n++] = t;
  }

  // intra_chroma_pred_mode for chroma_format_idc 2 / 3 (7.3.8.5, 8.4.3): one per prediction unit in 4:4:4; in 4:2:2 the mode goes
  // through Table 8-3 (as corrected: modeIdc 11 -> 12, 14 -> 17), packed here 6 bits per entry
  B200_HDN void chroma_modes_x(Cu& cu, int np) {
    const int cfmt = B200_SPC(chroma);
    B200_NOUNROLL for (int i = 0; i < (cfmt == 3 ? np : 1); i++) {
      int v = 4; if (dbin(CTX_CHROMA_PRED)) v = (int)dbits(2);
      int m;
      if (v == 4) m = cu.lmode[i]; else { m = B200_T(kChromaTab)[v]; if (m == cu.lmode[i]) m = 34; }
      if (cfmt == 2) {
        // {0,1,2,2,2,2,3,5,7,8 | 10,12,13,15,17,18,19,20,21,22 | 23,23,24,24,25,25,26,27,27,28 | 28,29,29,30,31}
        const unsigned long long w = m < 10 ? 0x207143082082040ull : (m < 20 ? 0x5955134913cd30aull : (m < 30 ? 0x71b6da6596185d7ull : 0x1f79d75cull));
        m = (int)((w >> (6 * (m % 10))) & 63ull);
      }
      cu.cmodes[i] = m;
    }
    cu.cmode = cu.cmodes[0];
  }

  // the 1 << (2 * l) cells of a square block (l = log2 of its side in cells) whose top-left cell is `m` in a map with `stride`
  // cells per row: `set` ? v : (cell | v)
  B200_HDI static void fill_cells(uint8_t* m, int stride, int l, uint8_t v, bool set) {
    B200_LANES_BEGIN();
    B200_LANE_FOR(k, 1 << (2 * l)) { uint8_t* p = m + (k >> l) * stride + (k & ((1 << l) - 1)); *p = set ? v : (uint8_t)(*p | v); }
    B200_LANES_END();
  }

  // -------- 7.3.8.5
  B200_HDI void coding_unit(int x0, int y0, int log2cb, int depth) {
    Cu cu; cu.x0 = x0; cu.y0 = y0; cu.log2cb = log2cb; cu.nxn = 0; cu.cmode = 0;
    const int n = 1 << log2cb;
    if (B200_SPC(tq_bypass)) {
      cu_bypass = dbin(CTX_TQ_BYPASS);
      // in-loop filters leave the samples of this unit unchanged (8.7.2.5.7 nDp / nDq = 0, 8.7.3 SaoTypeIdx = 0): bit 2 of the 8x8 cells
      if (cu_bypass) fill_cells(pb.edge8 + (y0 >> 3) * sp->w8 + (x0 >> 3), sp->w8, log2cb - 3, 4, false);
    }
    if (log2cb == B200_SPC(log2_min_cb)) cu.nxn = !dbin(CTX_PART_MODE);
    if (cu.nxn && log2cb == 3 && B200_SPC(log2_min_tb) > 2) { err = SYN_E_BITSTREAM; return; }
    if (B200_SPC(pcm) && !cu.nxn && log2cb >= sp->log2_min_pcm && log2cb <= sp->log2_max_pcm && cabac.terminate(stream)) { pcm_unit(x0, y0, log2cb, depth); return; }   // pcm_flag
    const int np = cu.nxn ? 4 : 1, pbs = cu.nxn ? n / 2 : n;
    int prev[4], mi[4] = {0, 0, 0, 0}, rem[4] = {0, 0, 0, 0};
    B200_NOUNROLL for (int i = 0; i < np; i++) prev[i] = dbin(CTX_PREV_INTRA);
    B200_NOUNROLL for (int i = 0; i < np; i++) { if (prev[i]) { mi[i] = dbypass(); if (mi[i]) mi[i] += dbypass(); } else rem[i] = (int)dbits(5); }
    B200_NOUNROLL for (int i = 0; i < np; i++) {
      const int px = x0 + (i & 1) * pbs, py = y0 + (i >> 1) * pbs;
      const int m = luma_mode(px, py, prev[i], mi[i], rem[i]);
      cu.lmode[i] = m;
      fill_cells(pb.ipm4 + (py >> 2) * sp->w4 + (px >> 2), sp->w4, log2cb - cu.nxn - 2, (uint8_t)m, true);
    }
    if (B200_SPC(chroma) >= 2) chroma_modes_x(cu, np);
    else if (B200_SPC(chroma)) {
      int v = 4; if (dbin(CTX_CHROMA_PRED)) v = (int)dbits(2);
      if (v == 4) cu.cmode = cu.lmode[0]; else { cu.cmode = B200_T(kChromaTab)[v]; if (cu.cmode == cu.lmode[0]) cu.cmode = 34; }
    }
    fill_cells(pb.cd8 + (y0 >> 3) * sp->w8 + (x0 >> 3), sp->w8, log2cb - 3, (uint8_t)depth, true);
    if (!B200_SPC(cu_qp_delta)) cur_qpy = ss->slice_qp; else derive_qpy(x0, y0);
    if (B200_SPC(chroma) >= 2) transform_tree_x(cu, sp->max_th_depth_intra + cu.nxn); else transform_tree(cu, sp->max_th_depth_intra + cu.nxn);
    fill_cells(reinterpret_cast<uint8_t*>(pb.qp8) + (y0 >> 3) * sp->w8 + (x0 >> 3), sp->w8, log2cb - 3, (uint8_t)(int8_t)cur_qpy, true);
    last_cu_qpy = cur_qpy;
  }

  // -------- 7.3.8.4
  // coding_quadtree (7.3.8.4) of one CTB, iteratively over minimum coding blocks in z-order (same walk as transform_tree)
  // Only the z-order position and the depth stay in registers across the calls of the walk: the CTB origin and the tree
  // size are read again from the decoder state (shared memory on the device, see run_substream) where they are needed.
  B200_HD inline int cq_levels() const { return sp->log2ctb - B200_SPC(log2_min_cb); }
  B200_HDI void coding_quadtree() {
    const int log2min = B200_SPC(log2_min_cb);
    B200_NOUNROLL for (int i = 0; i < (1 << (2 * cq_levels())) && !err;) {
      int depth = node_depth((unsigned)i, cq_levels());
      B200_NOUNROLL for (;;) {
        const int log2cb = sp->log2ctb - depth, n = 1 << log2cb;
        const int x0 = ctb_x0 + (zx((unsigned)i) << log2min), y0 = ctb_y0 + (zx((unsigned)i >> 1) << log2min);
        if (x0 >= sp->W || y0 >= sp->H) { i += 1 << (2 * (cq_levels() - depth)); break; }      // node outside the picture: not coded
        int split;
        if (x0 + n <= sp->W && y0 + n <= sp->H && log2cb > log2min) {
          int inc = 0;
          if (avail(x0 - 1, y0) && (int)pb.cd8[(y0 >> 3) * sp->w8 + ((x0 - 1) >> 3)] > depth) inc++;
          if (avail(x0, y0 - 1) && ld_cell(pb.cd8 + ((y0 - 1) >> 3) * sp->w8 + (x0 >> 3), y0 - 1) > depth) inc++;
          split = dbin(CTX_SPLIT_CU + inc);
        } else split = log2cb > log2min;
        if (B200_SPC(cu_qp_delta) && log2cb >= sp->qg_log2) {
          is_dqp_coded = 0; dqp_val = 0;
          if (!split || log2cb == sp->qg_log2) { if (first_qg) { qpy_prev_qg = ss->slice_qp; first_qg = 0; } else qpy_prev_qg = last_cu_qpy; }
        }
        if (split) { depth++; continue; }
        coding_unit(x0, y0, log2cb, depth);
        i += 1 << (2 * (cq_levels() - depth));
        break;
      }
    }
  }

  // One coding tree unit (7.3.8.2): SAO syntax + coding quadtree; fills its CtuInfo.
  B200_HDN void decode_ctb(int addr) {
    const int rx = addr % sp->wctb, ry = addr / sp->wctb;
    cur_ctb_x = rx; cur_ctb_y = ry;
    ctb_x0 = rx << sp->log2ctb; ctb_y0 = ry << sp->log2ctb;
    left_ok = rx > 0 && pb.ctu_slice[addr - 1] == (uint16_t)ss->slice_idx;
    up_ok = ry > 0 && pb.ctu_slice[addr - sp->wctb] == (uint16_t)ss->slice_idx;
    { // edges on the CTB boundary are filtered unless they are a slice boundary the current slice does not filter across, or a
      // tile boundary with loop_filter_across_tiles_enabled_flag = 0
      const SliceInfo& cs = pb.slices[ss->slice_idx];
      left_lf = left_ok; up_lf = up_ok;
      if (rx > 0 && !left_ok) { const SliceInfo& o = pb.slices[pb.ctu_slice[addr - 1]]; left_lf = (o.slice_id == cs.slice_id || cs.lf_across_slices) && (o.tile_id == cs.tile_id || cs.lf_across_tiles); }
      if (ry > 0 && !up_ok) { const SliceInfo& o = pb.slices[pb.ctu_slice[addr - sp->wctb]]; up_lf = (o.slice_id == cs.slice_id || cs.lf_across_slices) && (o.tile_id == cs.tile_id || cs.lf_across_tiles); } }
    CtuInfo& ci = pb.ctus[addr];
    ci.slice_idx = (uint16_t)ss->slice_idx;
    if (!B200_SPC(dense)) { tu_n = (uint32_t)addr * (uint32_t)sp->tu_slots; tu_cap = tu_n + (uint32_t)sp->tu_slots; coef_n = (uint32_t)addr * (uint32_t)sp->coef_slots; coef_cap = coef_n + (uint32_t)sp->coef_slots; }
    ctb_tu0 = tu_n;
    if (B200_SPC(sao_enabled)) parse_sao(rx, ry, ci);
    else for (int c = 0; c < 3; c++) { ci.sao[c].type = 0; ci.sao[c].band_or_class = 0; B200_NOUNROLL for (int k = 0; k < 4; k++) ci.sao[c].offset[k] = 0; }
    // 4x4 luma transform units only OR their edge bits: clear this CTB's flags first
    { const int l = sp->log2ctb - 3, b0x = rx << l, b0y = ry << l;
      B200_LANES_BEGIN();
      B200_LANE_FOR(k, 1 << (2 * l)) { const int y = b0y + (k >> l), x = b0x + (k & ((1 << l) - 1)); if (y < sp->h8 && x < sp->w8) pb.edge8[y * sp->w8 + x] = 0; }
      B200_LANES_END(); }
    coding_quadtree();
    CtuInfo& ce = pb.ctus[cur_ctb_y * sp->wctb + cur_ctb_x];        // (read again, like the quadtree's state)
    ce.tu_start = ctb_tu0; ce.tu_count = (uint16_t)(tu_n - ctb_tu0);
  }
};

typedef DecoderT<CfgRuntime> Decoder;

// Decodes one sub-stream.  `Sync` supplies wait_row(row, need) -- block until `need` CTBs of CTB row `row` are done --
// publish_row(row, done) and wait_substream(index); on the host (sequential order) they are no-ops.
template <class Cfg, class Sync>
// `d` is caller-provided storage: on the device it lives in SHARED memory -- a lone lane's local memory uses 4 bytes of
// every 128-byte line, so ~30 resident decoders with their state on the stack overflow L1 (measured: the SM's
// throughput stopped growing at 8 warps).
B200_HD int run_substream(DecoderT<Cfg>& d, const SeqParams& sp, const PicBuffers& pb, const Substream* all, int index, CtxPtr ctx, Sync& sync) {
  const Substream& ss = all[index];
  d.sp = &sp; d.pb = pb; d.ss = &ss; d.ctx = ctx; d.err = SYN_OK;
  d.is_dqp_coded = 0; d.dqp_val = 0; d.qpy_prev_qg = ss.slice_qp; d.last_cu_qpy = ss.slice_qp; d.first_qg = 1; d.cur_qpy = ss.slice_qp; d.cu_bypass = 0;
  d.tu_n = 0; d.coef_n = 0; d.tu_cap = 0; d.coef_cap = 0;
  if (B200_SPR(dense)) {                                             // host: continue the picture-wide cursors
    d.tu_n = sync.dense_tu; d.coef_n = sync.dense_coef; d.tu_cap = sync.dense_tu_cap; d.coef_cap = sync.dense_coef_cap;
  }
  const int rx0 = (int)(ss.ctb_begin % (uint32_t)sp.wctb), ry0 = (int)(ss.ctb_begin / (uint32_t)sp.wctb);
  // ---- context initialisation / synchronisation (9.3.1)
  if (ss.prev >= 0) {                                         // dependent slice segment: continue from the previous segment's end state
    sync.wait_substream(ss.prev);
    const uint8_t* st = pb.end_state + (size_t)ss.prev * CTX_STRIDE;
    load_contexts(ctx, st);
    d.last_cu_qpy = (int)(int8_t)B200_LD_SHARED(st + CTX_COUNT); d.first_qg = 0;
  }
  if (ss.init_contexts) init_contexts(ctx, ss.slice_qp);
  if (B200_SPR(wpp) && rx0 == 0 && (!ss.init_contexts || ss.prev >= 0) && ss.ctb_begin != ss.slice_addr_rs) {
    // first CTB of a row inside a slice: take the state stored after the 2nd CTB of the row above when that CTB is
    // available (same slice), otherwise initialise (or, for a dependent segment, keep the inherited state)
    const int xn = 1 << sp.log2ctb, yn = (ry0 - 1) << sp.log2ctb;
    bool tr = ry0 > 0 && xn < sp.W && pb.ctu_slice[(ry0 - 1) * sp.wctb + 1] == (uint16_t)ss.slice_idx;
    (void)yn;
    if (tr) { sync.wait_row(ry0 - 1, 2); load_contexts(ctx, pb.wpp_ctx + (size_t)(ry0 - 1) * CTX_STRIDE); }
    else if (ss.prev < 0) init_contexts(ctx, ss.slice_qp);
    d.first_qg = 1;
  }
  d.stream.d = pb.rbsp; d.stream.size = pb.rbsp_size;
  d.cabac.start(d.stream, ss.byte_begin);
  // From here on every parameter is read through `d` (and `sync`), never through the references above: on the device
  // both live in shared memory, and whatever is read again after a call into the decoder costs a shared-memory load per CTB
  // instead of a register for the whole call chain (its register count sets how many decoders fit on an SM).
  const bool tiles = B200_SPR(tiles) != 0;
  int rx = rx0, ry = ry0;
  B200_NOUNROLL for (uint32_t left = ss.ctb_end - ss.ctb_begin; left > 0; left--, rx++) {
    if (rx == (int)d.ss->tile_x1) { rx = (int)d.ss->tile_x0; ry++; }    // next row of the tile (of the picture without tiles)
    const uint32_t a = (uint32_t)ry * (uint32_t)d.sp->wctb + (uint32_t)rx;
    // split_cu_flag context / SAO merge-up read the CTB above (same column).  With tiles that CTB belongs to this very
    // sub-stream or is unavailable (another tile / slice), and rows are not produced in raster order: no hand-shake.
    if (ry > 0 && !tiles) sync.wait_row(ry - 1, rx + 1);
    if (B200_SPR(wpp) && rx == 0 && a != d.ss->ctb_begin) {
      // only reached without WPP sub-stream splitting (never: WPP rows are separate sub-streams); kept for safety
      d.first_qg = 1;
    }
    d.decode_ctb((int)a);
    if (d.err) break;
    rx = d.cur_ctb_x; ry = d.cur_ctb_y;
    if (B200_SPR(wpp) && rx == 1) store_contexts(d.ctx, d.pb.wpp_ctx + (size_t)ry * CTX_STRIDE);
    const int end = d.cabac.terminate(d.stream);                          // end_of_slice_segment_flag
    const bool last = left == 1;
    if (end != ((last && d.ss->last_of_segment) ? 1 : 0)) { d.err = SYN_E_BITSTREAM; break; }
    if (last && !d.ss->last_of_segment) { if (!d.cabac.terminate(d.stream)) { d.err = SYN_E_BITSTREAM; break; } }   // end_of_subset_one_bit
    if (!tiles) sync.publish_row(ry, rx + 1);
    if (B200_SPR(wpp) && rx == 1) sync.notify(d.ss->wake_ctb2);           // the row below may start (its context hand-over is stored)
    if (d.cabac.pos > d.pb.rbsp_size + 64u) { d.err = SYN_E_BITSTREAM; break; }
  }
  // end state for a dependent continuation + dense cursors
  { uint8_t* st = d.pb.end_state + (size_t)index * CTX_STRIDE; store_contexts(d.ctx, st); st[CTX_COUNT] = (uint8_t)(int8_t)d.last_cu_qpy; }
  if (B200_SPR(dense)) { sync.dense_tu = d.tu_n; sync.dense_coef = d.coef_n; }
  sync.end_bit_position = d.cabac.bit_position();
  sync.finish_substream(index, d.err);
  if (!d.err) sync.notify(d.ss->wake_end);
  return d.err;
}

}  // namespace syn
}  // namespace b200
