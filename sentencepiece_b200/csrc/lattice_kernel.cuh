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
//          end_nodes_ order: {id, score, begin character, the bytes of the character (UNK nodes)} --
//          and per position {A[pos], first node of end_nodes_[pos]}.  The backward sampling itself (std::exp,
//          std::discrete_distribution on std::mt19937) runs on the host, sentence after sentence on ONE generator:
//          that is what makes a seeded batch reproduce the reference's single-threaded stream bit for bit.
//   mode 1 (entropy):   H[pos] folded in a second pass over the nodes (A must be complete); -H[L] per sentence.
// A sentence the lane kernel cannot take (more than cap normalized bytes, or a lattice over node_cap nodes) goes on
// the deferred list (B.deferred, B.status[0]) for lattice_long_kernel, which computes the same outputs.
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
  uint32_t *status;                // [0] deferred sentences (shared with KBatch::status), [1] error, [2] output overflow
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
        lane_defer_long(B, sent, 0u);
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
        if (overflow) lane_defer_long(B, sent, n);
      }
      if (too_big || overflow) {
        // lattice_long_kernel writes this sentence's outputs
      } else if (mode == 1) {
        // ---- Lattice::CalculateEntropy (:266-291): H[end] += exp(tp) * (H[begin] + tp), tp = (theta * score + A[begin]) - A[end]
        float ent = 0.f;
        if (n != 0) {
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
        O.n_chars[sent] = L;
        if (n != 0) {
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
              O.nodes[ns + ecnt[e]++] = make_uint4(nd.x, nd.y, nd.z & 0xFFFFu, nd.w);
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

// ---- long-sentence path: one warp per sentence the lane kernel deferred (B.long_list: {sentence, normalized-byte
//      capacity}; B.long_scratch_off: its scratch slab), same outputs as lattice_lane_kernel, positions 32 bits wide.
//      The warp normalizes the sentence (normalize_tile), finds the character starts and walks the piece trie from
//      every start in parallel (a count pass, a scan, a write pass: nodes land in creation order); lane 0 folds A[end]
//      over the nodes in that order -- increasing begin position, the end_nodes_ order ForwardAlgorithm folds in --
//      and exports the lattice or folds H. ----
//   node [node_cap] uint4 {id, score bits, begin char, end char}; A, H (first the per-start node offsets), ecnt,
//   surf: [cap + 4] 4-byte words; text [cap + 16]
__host__ __device__ inline unsigned long long lattice_long_nodes(uint32_t cap, uint32_t mm1) {
  return static_cast<unsigned long long>(cap) * mm1 + 64ull;
}
__host__ __device__ inline unsigned long long lattice_long_bytes(uint32_t cap, uint32_t mm1) {
  const unsigned long long b = 16ull * lattice_long_nodes(cap, mm1) + 16ull * (cap + 4) + cap + 16;
  return (b + 255ull) & ~255ull;
}

__global__ void __launch_bounds__(256) lattice_long_kernel(const KModel M, const KBatch B, const LatticeOut O, uint32_t mm1,
                                                            float inv_theta, int mode) {
  const Tile T;
  const uint32_t lane = T.lane;
  const uint32_t root = __ldg(&M.trie_node2[0]).x;
  const uint32_t warps = blockDim.x >> 5;
  for (uint32_t w = blockIdx.x * warps + (threadIdx.x >> 5); w < B.long_n; w += gridDim.x * warps) {
    const uint32_t sent = B.long_list[2 * w], cap = B.long_list[2 * w + 1];
    const unsigned long long node_cap = lattice_long_nodes(cap, mm1);
    uint8_t *sp = B.long_scratch + B.long_scratch_off[w];
    uint4 *node = reinterpret_cast<uint4 *>(sp); sp += 16ull * node_cap;
    float *A = reinterpret_cast<float *>(sp); sp += 4ull * (cap + 4);
    float *H = reinterpret_cast<float *>(sp); sp += 4ull * (cap + 4);
    uint32_t *ecnt = reinterpret_cast<uint32_t *>(sp); sp += 4ull * (cap + 4);
    uint32_t *surf = reinterpret_cast<uint32_t *>(sp); sp += 4ull * (cap + 4);
    uint8_t *text = sp;
    uint32_t *nstart = reinterpret_cast<uint32_t *>(H);

    TileMem tm{};
    tm.text = text;
    tm.ncap = cap;
    const unsigned long long off = B.offsets[sent];
    const uint32_t n = normalize_tile<false>(M, T, B.bytes + off, static_cast<uint32_t>(B.offsets[sent + 1] - off), tm).n;
    if (n > cap) {  // the slab was sized from an upper bound of the normalized length
      if (lane == 0) atomicOr(O.status + 1, 8u);
      continue;
    }
    uint32_t L = 0, nn = 0;
    if (n != 0) {
      L = long_char_starts(text, n, surf, lane);
      auto text_byte = [&](uint32_t k) -> uint32_t { return text[k]; };
      // ---- Model::PopulateNodes: count the nodes of every start, then write them at their offsets ----
      for (uint32_t b0 = 0; b0 < L; b0 += 32) {
        const uint32_t bp = b0 + lane;
        uint32_t cnt = 0;
        if (bp < L) {
          const bool single = populate_from(M, text_byte, root, surf, bp, n, [&](uint32_t, uint32_t, float) { ++cnt; return true; });
          cnt += single ? 0u : 1u;
        }
        const uint32_t incl = T.incl_scan(cnt);
        if (bp < L) nstart[bp] = nn + incl - cnt;
        nn += T.shfl(incl, 31);
      }
      if (nn > node_cap) {  // more matches per start than the model's trie reports
        if (lane == 0) atomicOr(O.status + 1, 16u);
        continue;
      }
      for (uint32_t bp = lane; bp < L; bp += 32) {
        uint32_t k = nstart[bp];
        const bool single = populate_from(M, text_byte, root, surf, bp, n, [&](uint32_t length, uint32_t v, float sc) {
          node[k++] = make_uint4(static_cast<uint32_t>(__ldg(M.trie_id + v)), __float_as_uint(sc), bp, bp + length);
          return true;
        });
        if (!single) node[k] = make_uint4(static_cast<uint32_t>(M.unk_id), __float_as_uint(M.unk_score), bp, bp + 1);
      }
      for (uint32_t p = lane; p <= L + 1; p += 32) { A[p] = __uint_as_float(kLatticeUnset); ecnt[p] = 0; H[p] = 0.f; }
      __syncwarp();
      if (lane == 0) {
        // ---- Lattice::ForwardAlgorithm, arithmetic of lattice_lane_kernel ----
        A[0] = 0.f;
        for (uint32_t i = 0; i < nn; ++i) {
          const uint4 nd = node[i];
          ecnt[nd.w] += 1;
          const float y = __fadd_rn(__fmul_rn(inv_theta, __uint_as_float(nd.y)), A[nd.z]);
          const float cur = A[nd.w];
          A[nd.w] = __float_as_uint(cur) == kLatticeUnset ? y : lattice_log_sum_exp(cur, y);
        }
        if (mode == 1) {
          // ---- Lattice::CalculateEntropy; exp(tp) rounded from double, as close to the reference's std::exp(float)
          //      as the device gets: over a long sentence expf's last-place errors would add up in H ----
          for (uint32_t i = 0; i < nn; ++i) {
            const uint4 nd = node[i];
            const float tp = __fsub_rn(__fadd_rn(__fmul_rn(inv_theta, __uint_as_float(nd.y)), A[nd.z]), A[nd.w]);
            const float ex = static_cast<float>(exp(static_cast<double>(tp)));
            H[nd.w] = __fadd_rn(H[nd.w], __fmul_rn(ex, __fadd_rn(H[nd.z], tp)));
          }
        }
      }
      __syncwarp();
    }
    if (mode == 1) {
      if (lane == 0) O.entropy[sent] = n != 0 ? -H[L] : 0.f;
      continue;
    }
    // ---- export, as lattice_lane_kernel ----
    unsigned long long ns = 0, ps = 0;
    bool room = true;
    if (lane == 0) {
      O.n_chars[sent] = L;
      if (n != 0) {
        ns = atomicAdd(O.cursor, static_cast<unsigned long long>(nn));
        ps = atomicAdd(O.cursor + 1, static_cast<unsigned long long>(L + 2));
        room = ns + nn <= O.node_cap && ps + L + 2 <= O.pos_cap;
        if (!room) atomicOr(O.status + 2, 1u);
      }
      O.node_start[sent] = ns;
      O.pos_start[sent] = ps;
    }
    if (n == 0 || !__shfl_sync(0xFFFFFFFFu, room, 0)) continue;
    ps = __shfl_sync(0xFFFFFFFFu, ps, 0);
    ns = __shfl_sync(0xFFFFFFFFu, ns, 0);
    uint32_t run = 0;  // exclusive prefix of the per-end counts
    for (uint32_t p0 = 0; p0 <= L; p0 += 32) {
      const uint32_t p = p0 + lane;
      const uint32_t cnt = p <= L ? ecnt[p] : 0u;
      const uint32_t incl = T.incl_scan(cnt);
      if (p <= L) {
        O.pos[ps + p] = make_uint2(__float_as_uint(A[p]), run + incl - cnt);
        ecnt[p] = run + incl - cnt;
      }
      run += T.shfl(incl, 31);
    }
    if (lane == 0) {
      O.pos[ps + L + 1] = make_uint2(0u, run);
      for (uint32_t i = 0; i < nn; ++i) {  // stable counting sort by end position
        const uint4 nd = node[i];
        uint32_t chb = 0;
        if (static_cast<int32_t>(nd.x) == M.unk_id)
          for (uint32_t k = surf[nd.z]; k < surf[nd.z + 1]; ++k) chb |= static_cast<uint32_t>(text[k]) << (8u * (k - surf[nd.z]));
        O.nodes[ns + ecnt[nd.w]++] = make_uint4(nd.x, nd.y, nd.z, chb);
      }
    }
    __syncwarp();
  }
}

}  // namespace spm_b200
#endif
