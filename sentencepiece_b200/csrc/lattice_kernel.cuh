// lattice_kernel.cuh -- full-lattice operations of unigram models (SURVEY 8f item 1), one sentence per lane.
//
// Reference: Lattice::SetSentence (src/unigram_model.cc:113-146), Model::PopulateNodes (:547-596),
// Lattice::ForwardAlgorithm (:200-217) with LogSumExp (:47-59), Lattice::CalculateEntropy (:266-291) and the
// candidate lists Lattice::Sample (:511-542) draws from.
//
// alpha[node] of the reference only depends on the character position the node BEGINS at (every node beginning at
// pos folds the same end_nodes_[pos] list in the same order), so the kernel keeps one float A[pos] per position.
// end_nodes_[pos] is ordered by begin position (PopulateNodes walks begin positions left to right), which is also
// the order in which this kernel creates nodes: A[end] is folded as nodes are created ("push" form), A[begin] is
// final by then because every node ending at `begin` starts earlier.  Arithmetic as in the reference: float
// product inv_theta * score, float sum with A[begin], LogSumExp = vmax + log(exp(double(vmin - vmax)) + 1.0)
// evaluated in double and rounded to float (CUDA's double exp / log are within 1 ulp of glibc's, so the float
// result is identical except for astronomically rare double-rounding ties; the parity tests compare bit for bit).
//
//   mode 0 (sampling):  per sentence the kernel exports the lattice -- nodes sorted by end position, in
//          end_nodes_ order: {id, score, begin | end << 16 (characters), the bytes of the character (UNK nodes)} --
//          and per position {A[pos], first node of end_nodes_[pos]}.  The backward sampling itself (std::exp,
//          std::discrete_distribution on std::mt19937) runs on the host, sentence after sentence on ONE generator:
//          that is what makes a seeded batch reproduce the reference's single-threaded stream bit for bit.
//   mode 1 (entropy):   H[pos] folded in a second pass over the nodes (A must be complete); -H[L] per sentence.
#ifndef SPM_B200_LATTICE_KERNEL_CUH_
#define SPM_B200_LATTICE_KERNEL_CUH_

#include "lane_kernel.cuh"

namespace spm_b200 {

struct LatticeGeom {
  uint32_t cap;       // normalized bytes per sentence
  uint32_t node_cap;  // lattice nodes per sentence
};
// per-lane scratch: surf u16[cap+4], A f32[cap+4], H f32[cap+4], ecnt u32[cap+4], node uint4[node_cap]
__host__ __device__ inline unsigned long long lattice_lane_bytes(const LatticeGeom &g) {
  unsigned long long b = 16ull * g.node_cap + (4ull + 4ull + 4ull) * (g.cap + 4) + 2ull * (g.cap + 4);
  return (b + 15ull) & ~15ull;
}

struct LatticeOut {
  uint4 *nodes;                    // packed node records of all sentences (mode 0)
  uint2 *pos;                      // packed {A bits, end_off} records, L + 2 per sentence (mode 0)
  unsigned long long node_cap, pos_cap;
  unsigned long long *cursor;      // [0] nodes, [1] pos records
  unsigned long long *node_start;  // [n]
  unsigned long long *pos_start;   // [n]
  uint32_t *n_chars;               // [n] L (0: empty normalized text)
  float *entropy;                  // [n] (mode 1)
  uint32_t *status;                // [1] error, [2] output overflow, [3] capacity exceeded (unsupported)
};

constexpr uint32_t kLatticeUnset = 0x7FC00001u;  // A[pos] not folded yet (a NaN pattern no sum can produce)

__device__ __forceinline__ float lattice_log_sum_exp(float x, float y) {  // unigram_model.cc:47-59, init_mode == false
  const float vmin = fminf(x, y), vmax = fmaxf(x, y);
  if (vmax > __fadd_rn(vmin, 50.f)) return vmax;
  return static_cast<float>(static_cast<double>(vmax) + log(exp(static_cast<double>(__fsub_rn(vmin, vmax))) + 1.0));
}

__global__ void __launch_bounds__(512, 1) lattice_lane_kernel(const KModel M, const KBatch B, const LatticeOut O,
                                                               uint8_t *text_slabs, uint8_t *scratch,
                                                               const LatticeGeom G, float inv_theta, int mode) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint32_t *s_tab = reinterpret_cast<uint32_t *>(smem);
  fill_lane_tables(M, s_tab);
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warp_global = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const LaneCtx c = lane_ctx(s_tab, text_slabs, G.cap, warp_global, lane);
  uint8_t *sp = scratch + (static_cast<size_t>(warp_global) * 32 + lane) * lattice_lane_bytes(G);
  uint4 *node = reinterpret_cast<uint4 *>(sp); sp += 16ull * G.node_cap;
  float *A = reinterpret_cast<float *>(sp); sp += 4ull * (G.cap + 4);
  float *H = reinterpret_cast<float *>(sp); sp += 4ull * (G.cap + 4);
  uint32_t *ecnt = reinterpret_cast<uint32_t *>(sp); sp += 4ull * (G.cap + 4);
  uint16_t *surf = reinterpret_cast<uint16_t *>(sp);
  const uint32_t root = __ldg(&M.trie_node2[0]).x;

  uint32_t first = 0;
  while (lane_claim_group(B, lane, &first)) {
    if (first + lane < B.n) {
      const uint32_t sent = B.order ? B.order[first + lane] : first + lane;
      uint32_t n;
      const bool too_big = !lane_k1(M, B, c, sent, G.cap, &n);
      uint32_t L = 0;
      bool overflow = false;
      uint32_t nn = 0;
      if (too_big) {
        atomicOr(O.status + 3, 1u);
      } else if (n != 0) {
        // ---- Lattice::SetSentence ----
        for (uint32_t p = 0; p < n;) {
          uint32_t mb = one_char_len(lane_text_byte_plain(c, p));
          if (mb > n - p) mb = n - p;
          surf[L] = static_cast<uint16_t>(p);
          A[L] = __uint_as_float(kLatticeUnset);
          ecnt[L] = 0;
          ++L;
          p += mb;
        }
        surf[L] = static_cast<uint16_t>(n);
        A[L] = __uint_as_float(kLatticeUnset);
        ecnt[L] = 0;
        ecnt[L + 1] = 0;
        A[0] = 0.f;  // nodes beginning at 0 fold {BOS}: LogSumExp(., 0 * 0 + 0, init) = 0
        // ---- Model::PopulateNodes with Lattice::ForwardAlgorithm folded in ----
        for (uint32_t bp = 0; bp < L && !overflow; ++bp) {
          const float a = A[bp];
          auto add_node = [&](uint32_t ep, int32_t id, float sc, uint32_t chbytes) -> bool {
            if (nn >= G.node_cap) { overflow = true; return false; }
            node[nn++] = make_uint4(static_cast<uint32_t>(id), __float_as_uint(sc), bp | (ep << 16), chbytes);
            ecnt[ep] += 1;
            const float y = __fadd_rn(__fmul_rn(inv_theta, sc), a);
            const float cur = A[ep];
            A[ep] = __float_as_uint(cur) == kLatticeUnset ? y : lattice_log_sum_exp(cur, y);
            return true;
          };
          const bool has_single = lane_populate_from(M, c, root, surf, bp, n, [&](uint32_t length, uint32_t v, float sc) {
            return add_node(bp + length, __ldg(M.trie_id + v), sc, 0u);
          });
          if (!has_single && !overflow) {
            uint32_t chb = 0;
            for (uint32_t k = surf[bp]; k < surf[bp + 1]; ++k) chb |= lane_text_byte_plain(c, k) << (8u * (k - surf[bp]));
            add_node(bp + 1, M.unk_id, M.unk_score, chb);
          }
        }
        if (overflow) atomicOr(O.status + 3, 1u);
      }
      if (mode == 1) {
        // ---- Lattice::CalculateEntropy (:266-291): H[end] += exp(tp) * (H[begin] + tp), tp = (theta * score + A[begin]) - A[end]
        float ent = 0.f;
        if (n != 0 && !overflow && !too_big) {
          for (uint32_t p = 0; p <= L; ++p) H[p] = 0.f;
          for (uint32_t i = 0; i < nn; ++i) {
            const uint4 nd = node[i];
            const uint32_t b = nd.z & 0xFFFFu, e = nd.z >> 16;
            const float tp = __fsub_rn(__fadd_rn(__fmul_rn(inv_theta, __uint_as_float(nd.y)), A[b]), A[e]);
            H[e] = __fadd_rn(H[e], __fmul_rn(expf(tp), __fadd_rn(H[b], tp)));
          }
          // EOS folds end_nodes_[L] with tp = 0 * ... : handled above through H[L]; the reference adds, for rnode = EOS,
          // the contributions of the nodes ending at L, which is exactly H[L]
          ent = -H[L];
        }
        O.entropy[sent] = ent;
      } else {
        // ---- export: nodes in end_nodes_ order (stable counting sort by end position) + per-position records ----
        O.n_chars[sent] = (too_big || overflow) ? 0u : L;
        if (n != 0 && !overflow && !too_big) {
          const unsigned long long ns = atomicAdd(O.cursor, static_cast<unsigned long long>(nn));
          const unsigned long long ps = atomicAdd(O.cursor + 1, static_cast<unsigned long long>(L + 2));
          O.node_start[sent] = ns;
          O.pos_start[sent] = ps;
          if (ns + nn > O.node_cap || ps + L + 2 > O.pos_cap) {
            atomicOr(O.status + 2, 1u);
          } else {
            // exclusive prefix of the per-end counts; position 0 holds BOS only (no record)
            uint32_t run = 0;
            for (uint32_t p = 0; p <= L; ++p) {
              const uint32_t cnt = ecnt[p];
              O.pos[ps + p] = make_uint2(__float_as_uint(A[p]), run);
              ecnt[p] = run;
              run += cnt;
            }
            O.pos[ps + L + 1] = make_uint2(0u, run);
            for (uint32_t i = 0; i < nn; ++i) {
              const uint4 nd = node[i];
              const uint32_t e = nd.z >> 16;
              O.nodes[ns + ecnt[e]++] = nd;
            }
          }
        } else {
          O.node_start[sent] = 0;
          O.pos_start[sent] = 0;
        }
      }
    }
    __syncwarp();
  }
}

}  // namespace spm_b200
#endif
