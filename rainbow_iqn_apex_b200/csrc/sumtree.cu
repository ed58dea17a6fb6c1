// Device-resident prioritized-replay sum-tree and frame store (reference rainbowiqn/redis_memory.py).
//
// The reference keeps the tree as Redis string keys "priorities:<i>" (decimal strings parsed to
// float64) and spends one network round trip per tree level; here the 2C-1 float64 nodes live in HBM
// (implicit heap, leaf of data index d at d + C - 1) and every operation is one or two launches.
// All arithmetic is float64 in the reference's exact order, so indices and node values are bit-exact:
//   * descent:  `if value <= left: go left else value -= left; go right`, non-power-of-two guard
//               (redis_memory.py:205-229)
//   * update:   old leaves read first (duplicates see the same old), diff = new - old; every ancestor
//               gets `+= diff` sequentially in batch order; index 0 skipped on the way up and the root
//               finally receives numpy's pairwise np.sum(diffs) (redis_memory.py:94-105,139-151)
//   * valid-index shift away from actor write heads (redis_memory.py:242-264)
#include <climits>

#include "common.cuh"
#include "../../include/riqn_b200.h"

namespace riqn {

// ------------------------------------------------------------------------------------------------
// Sampling
// ------------------------------------------------------------------------------------------------
// samples[i] = a + (b - a) * u_i, a = i*seg, b = (i+1)*seg (CPython random.uniform), then shuffled
// (redis_memory.py:276-287).  Single CTA; thread 0 runs the Fisher-Yates shuffle in shared memory.
__global__ void stratified_kernel(int n, uint64_t seed, uint64_t stream, const double* __restrict__ tree,
                                  double* __restrict__ values, const riqn_dyn_state* __restrict__ dyn) {
  if (dyn) stream += dyn->rng_offset;
  // the shuffle: stratum s goes to output slot rank(key_s), keys = Philox draws (ties broken by index)
  extern __shared__ uint32_t keys[];
  const double seg = tree[0] / (double)n;
  for (int i = threadIdx.x; i < n; i += blockDim.x) keys[i] = Philox::draw(seed, stream ^ 0x5bd1e995ull, (uint64_t)i).x;
  __syncthreads();
  for (int s = threadIdx.x; s < n; s += blockDim.x) {
    const uint32_t me = keys[s];
    int rank = 0;
    for (int j = 0; j < n; ++j) rank += (keys[j] < me) || (keys[j] == me && j < s);
    const uint4 r = Philox::draw(seed, stream, (uint64_t)s);
    const double a = (double)s * seg, b = (double)(s + 1) * seg;
    values[rank] = __dadd_rn(a, __dmul_rn(b - a, Philox::u01d(r.x, r.y)));   // a + (b-a)*u, no FMA contraction
  }
}

// One warp per query.  The warp prefetches the whole 5-level subtree under the current node (62 nodes,
// two coalesced 8-byte loads per lane), then walks it with shuffles: 5 levels per dependent memory
// round trip instead of 1, using exactly the reference's stored node values and comparison order.
// HZ: the shift's n_step is this step's hz->n_step, read on the device and kept in 1..n_step (the by-value n_max).
template <bool HZ>
__global__ void sumtree_sample_kernel(int n, long C, int actor_cap, const double* __restrict__ tree,
                                      const double* __restrict__ values, const int64_t* __restrict__ index_actor,
                                      int history, int n_step, const riqn_horizon_state* __restrict__ hz,
                                      int64_t* __restrict__ tree_idx, int64_t* __restrict__ data_idx,
                                      double* __restrict__ priorities) {
  if constexpr (HZ) n_step = min(max(hz->n_step, 1), n_step);
  const int lane = threadIdx.x & 31;
  const long q = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (q >= n) return;
  const long n_nodes = 2 * C - 1;
  long idx = 0;
  double value = values[q];
  while (2 * idx + 1 < n_nodes) {
    // relative level l (1..5) under idx holds nodes (idx+1)*2^l - 1 + [0, 2^l)
    // lane j loads: slot j  -> levels 1..4 packed (30 nodes: offsets 0..29), slot 32+j -> level 5
    double lo = 0.0, hi = 0.0;
    {
      // packed index p in [0,30): level l = floor(log2(p+2)), pos = p + 2 - 2^l
      const int p = lane;
      if (p < 30) {
        const int l = 31 - __clz(p + 2);
        const long node = ((idx + 1) << l) - 1 + (p + 2 - (1 << l));
        if (node < n_nodes) lo = tree[node];
      }
      const long node5 = ((idx + 1) << 5) - 1 + lane;
      if (node5 < n_nodes) hi = tree[node5];
    }
    int pos = 0;  // position within the current relative level
#pragma unroll
    for (int l = 1; l <= 5; ++l) {
      const long left = 2 * idx + 1;
      if (left >= n_nodes) break;  // warp-uniform
      const int lpos = 2 * pos;    // left child position in level l
      double left_sum;
      if (l < 5) left_sum = __shfl_sync(0xffffffffu, lo, (1 << l) - 2 + lpos);
      else left_sum = __shfl_sync(0xffffffffu, hi, lpos);
      if (value <= left_sum) { idx = left; pos = lpos; }
      else { idx = left + 1; value = value - left_sum; pos = lpos + 1; }
    }
  }
  if (lane == 0) {
    // transform_to_valid_tree_indexes                                  redis_memory.py:242-264
    long d = idx - C + 1;
    const long actor = d / actor_cap;
    const long dist = (d % actor_cap) - index_actor[actor];
    if (dist >= 0 && dist <= history) {
      long t = (d + history - dist + 1) % actor_cap;
      d = t + actor * actor_cap;
    } else if (dist < 0 && dist >= -n_step) {
      long t = (d - n_step - dist - 1) % actor_cap;
      if (t < 0) t += actor_cap;  // python modulo
      d = t + actor * actor_cap;
    }
    const long ti = d + C - 1;
    tree_idx[q] = ti;
    data_idx[q] = d;
    priorities[q] = tree[ti];
  }
}

// w = (capacity * p / p_total)^-beta / max(w)                           redis_memory.py:465-475
// Non-positive priorities fall back to the uniform 1/capacity (redis_memory.py:446-456); their count
// is reported so the host can apply the reference's resample-first policy if it wants to.
__global__ void is_weights_kernel(int n, const double* __restrict__ tree, const double* __restrict__ priorities,
                                  double capacity, double beta, double* __restrict__ w64, float* __restrict__ w32,
                                  int* __restrict__ n_nonpositive, const riqn_dyn_state* __restrict__ dyn) {
  if (dyn) { capacity = dyn->is_capacity; beta = dyn->is_beta; }
  __shared__ double red[32];
  __shared__ int cnt;
  if (threadIdx.x == 0) cnt = 0;
  __syncthreads();
  const double p_total = tree[0];
  double mx = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    double p = priorities[i];
    if (p <= 0.0) { p = 1.0 / capacity; atomicAdd(&cnt, 1); }
    const double w = pow(capacity * (p / p_total), -beta);
    w64[i] = w;
    mx = fmax(mx, w);
  }
  for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x < 32) {
    mx = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.0;
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (threadIdx.x == 0) red[0] = mx;
  }
  __syncthreads();
  mx = red[0];
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const double w = w64[i] / mx;
    w64[i] = w;
    w32[i] = (float)w;
  }
  if (threadIdx.x == 0 && n_nonpositive) *n_nonpositive = cnt;
}

// ------------------------------------------------------------------------------------------------
// Update
// ------------------------------------------------------------------------------------------------
// priorities = np.power(loss_f32, float32(omega))  (redis_memory.py:560) evaluated as a correctly
// rounded float: double pow then one rounding.  exponent < 0 sentinel => priorities passed through.
// DEMO: DQfD's demonstration bonus, p = fl(p + bonus) on the leaves idx >= demo_leaf, after the power.
template <bool DEMO>
__global__ void update_prepare_kernel(int n, const double* __restrict__ tree, const int64_t* __restrict__ idx,
                                      const float* __restrict__ loss, float exponent, int apply_pow,
                                      float* __restrict__ new_pri, double* __restrict__ diff,
                                      double* __restrict__ max_priority, int64_t demo_leaf, float bonus) {
  __shared__ float red[32];
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    float p = loss[j];
    if (apply_pow) p = (float)pow((double)p, (double)exponent);
    if constexpr (DEMO) {
      if (idx[j] >= demo_leaf) p = __fadd_rn(p, bonus);
    }
    new_pri[j] = p;
    diff[j] = (double)p - tree[idx[j]];
    mx = fmaxf(mx, p);
  }
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x < 32) {
    mx = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : -INFINITY;
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (threadIdx.x == 0 && (double)mx > *max_priority) *max_priority = (double)mx;   // :150-151
  }
}

// numpy pairwise summation (np.sum of a contiguous float64 vector == 0 + pairwise(a, n)): blocks of <= 128
// elements are summed with 8 interleaved accumulators, larger ranges split at n/2 rounded down to a multiple
// of 8 and the two halves added.  Iterative post-order walk of that recursion (no device stack needed).
__device__ __forceinline__ double np_block_sum(const double* a, int n) {
  if (n < 8) {
    double r = 0.0;
    for (int i = 0; i < n; ++i) r += a[i];
    return r;
  }
  double r[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) r[k] = a[k];
  int i = 8;
  for (; i < n - (n % 8); i += 8) {
#pragma unroll
    for (int k = 0; k < 8; ++k) r[k] += a[i + k];
  }
  double res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
  for (; i < n; ++i) res += a[i];
  return res;
}

// The recursion walk; leaf(off, len, ordinal) supplies the sum of the ordinal-th block (left to right).
template <typename Leaf>
__device__ __forceinline__ double np_pairwise_walk(int n, Leaf leaf) {
  int off[24], len[24], stage[24];
  double left[24];
  int sp = 0, ordinal = 0;
  off[0] = 0; len[0] = n; stage[0] = 0; sp = 1;
  double ret = 0.0;
  while (sp > 0) {
    const int t = sp - 1;
    if (len[t] <= 128) {
      ret = leaf(off[t], len[t], ordinal++);
      --sp;
      // hand the value to the ancestors that are waiting for it
      while (sp > 0) {
        const int p = sp - 1;
        if (stage[p] == 1) {  // left half done -> start the right half
          left[p] = ret;
          stage[p] = 2;
          int n2 = len[p] / 2;
          n2 -= n2 % 8;
          off[sp] = off[p] + n2; len[sp] = len[p] - n2; stage[sp] = 0;
          ++sp;
          break;
        }
        ret = left[p] + ret;  // stage 2: both halves done
        --sp;
      }
    } else {
      int n2 = len[t] / 2;
      n2 -= n2 % 8;
      stage[t] = 1;
      off[sp] = off[t]; len[sp] = n2; stage[sp] = 0;
      ++sp;
    }
  }
  return ret;
}

__device__ double np_pairwise_sum(const double* a, int n) {
  return np_pairwise_walk(n, [a](int off, int len, int) { return np_block_sum(a + off, len); });
}

// The same sum computed by a whole CTA with the SAME operation order: thread 0 lists the <= 128-element blocks, the 8
// interleaved accumulators of every block run on separate threads, and thread 0 combines the block sums along the
// recursion.  lo / ll (block offsets / lengths), racc (8 per block), bsum (1 per block): shared scratch for
// n / 64 + 2 blocks.  Returns the sum on thread 0.
__device__ double np_pairwise_sum_cta(const double* a, int n, int* lo, int* ll, double* racc, double* bsum, int* n_blocks) {
  if (threadIdx.x == 0) {
    int cnt = 0;
    np_pairwise_walk(n, [&](int off, int len, int) { lo[cnt] = off; ll[cnt] = len; ++cnt; return 0.0; });
    *n_blocks = cnt;
  }
  __syncthreads();
  const int nb = *n_blocks;
  for (int t = threadIdx.x; t < nb * 8; t += blockDim.x) {
    const int blk = t >> 3, k = t & 7, len = ll[blk];
    const double* x = a + lo[blk];
    if (len >= 8) {
      double r = x[k];
      for (int i = 8; i < len - (len % 8); i += 8) r += x[i + k];
      racc[t] = r;
    }
  }
  __syncthreads();
  for (int blk = threadIdx.x; blk < nb; blk += blockDim.x) {
    const int len = ll[blk];
    const double* x = a + lo[blk];
    double res;
    if (len < 8) {
      res = 0.0;
      for (int i = 0; i < len; ++i) res += x[i];
    } else {
      const double* r = racc + blk * 8;
      res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
      for (int i = len - (len % 8); i < len; ++i) res += x[i];
    }
    bsum[blk] = res;
  }
  __syncthreads();
  double ret = 0.0;
  if (threadIdx.x == 0) ret = np_pairwise_walk(n, [bsum](int, int, int ordinal) { return bsum[ordinal]; });
  return ret;
}

// gridDim.y CTAs per tree depth d >= 1 (blockIdx.x = d - 1) share the batch entries; the last x-row does the root.  For a node X at depth d
// the reference applies, level by level, first the diffs of batch entries whose leaf is fewer parent steps
// away (the shallower leaves of a non-power-of-two tree), then the deeper ones, each group in batch order
// (redis_memory.py:94-105).  The warp of the first batch entry that touches X replays exactly that sequence of
// float64 adds, so every node is written once.
__global__ void update_propagate_kernel(int n, int max_depth, double* __restrict__ tree,
                                        const int64_t* __restrict__ idx, const double* __restrict__ diff) {
  extern __shared__ unsigned char smem_raw[];
  int64_t* node = reinterpret_cast<int64_t*>(smem_raw);
  double* sd = reinterpret_cast<double*>(node + n);
  int* steps = reinterpret_cast<int*>(sd + n);
  if ((int)blockIdx.x == max_depth) {  // root: tree[0] += np.sum(diffs)
    if (blockIdx.y != 0) return;
    for (int j = threadIdx.x; j < n; j += blockDim.x) sd[j] = diff[j];
    __syncthreads();
    __shared__ int p_lo[66], p_ll[66], p_nb;
    __shared__ double p_racc[66 * 8], p_bsum[66];
    const double tot = np_pairwise_sum_cta(sd, n, p_lo, p_ll, p_racc, p_bsum, &p_nb);
    if (threadIdx.x == 0) tree[0] = tree[0] + (0.0 + tot);
    return;
  }
  const int d = blockIdx.x + 1;
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    const int64_t leaf = idx[j];
    const int depth = 63 - __clzll((unsigned long long)(leaf + 1));  // floor(log2(leaf + 1))
    const int st = depth - d;                                        // parent steps from the leaf to depth d
    node[j] = st >= 0 ? ((leaf + 1) >> st) - 1 : -1;
    steps[j] = st;
    sd[j] = diff[j];
  }
  __syncthreads();
  // One warp per batch entry j (the entries of one depth are shared out over the warps of gridDim.y CTAs; every CTA
  // still holds all n entries in shared memory).  The 32 lanes scan the batch 128 entries per step: first occurrence
  // of j's node and the range of parent-step counts among its hits, reduced with redux.sync.  The owning warp then
  // replays the float64 adds in the reference's order; the hit masks come from ballots, so every lane walks the
  // same bits and carries the same accumulator (no divergence, shared-memory reads are broadcasts).
  constexpr unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  for (int j = blockIdx.y * wpb + warp; j < n; j += gridDim.y * wpb) {
    const int64_t me = node[j];
    if (me <= 0) continue;
    int first = n, smin = INT_MAX, smax = INT_MIN;
    for (int k0 = 0; k0 < n; k0 += 128) {
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int k = k0 + 32 * u + lane;
        if (k < n && node[k] == me) {
          const int st = steps[k];
          first = min(first, k);
          smin = min(smin, st);
          smax = max(smax, st);
        }
      }
      // an earlier entry owns this node: nothing more to learn from the rest of the batch
      if (__any_sync(FULL, first < j)) break;
    }
    first = __reduce_min_sync(FULL, first);
    if (first != j) continue;
    smin = __reduce_min_sync(FULL, smin);
    smax = __reduce_max_sync(FULL, smax);
    double acc = tree[me];
    for (int s = smin; s <= smax; ++s) {
      for (int k0 = j & ~127; k0 < n; k0 += 128) {         // no hit below j (j is the first occurrence)
        unsigned m[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int k = k0 + 32 * u + lane;
          m[u] = __ballot_sync(FULL, k < n && node[k] == me && steps[k] == s);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          unsigned mm = m[u];
          while (mm) {
            const int b = __ffs(mm) - 1;
            mm &= mm - 1;
            acc += sd[k0 + 32 * u + b];
          }
        }
      }
    }
    if (lane == 0) tree[me] = acc;
  }
}

// ------------------------------------------------------------------------------------------------
// Frame store
// ------------------------------------------------------------------------------------------------
constexpr int FRAME_BYTES = 84 * 84;  // 7056 = 441 * 16

// append_actor_buffer, frame half: slots (start + i) % actor_cap + actor*actor_cap   (:159-165,174-199)
__global__ void replay_append_kernel(int n, int actor_cap, int id_actor, int start, const uint8_t* __restrict__ frames,
                                     const int32_t* __restrict__ timestep, const int32_t* __restrict__ action,
                                     const float* __restrict__ reward, const uint8_t* __restrict__ nonterminal,
                                     uint8_t* __restrict__ s_frames, int32_t* __restrict__ s_timestep,
                                     int32_t* __restrict__ s_action, float* __restrict__ s_reward,
                                     uint8_t* __restrict__ s_nonterminal) {
  const int i = blockIdx.x;
  const long slot = (long)((start + i) % actor_cap) + (long)id_actor * actor_cap;
  const uint4* src = reinterpret_cast<const uint4*>(frames + (long)i * FRAME_BYTES);
  uint4* dst = reinterpret_cast<uint4*>(s_frames + slot * FRAME_BYTES);
  for (int t = threadIdx.x; t < FRAME_BYTES / 16; t += blockDim.x) dst[t] = src[t];
  if (threadIdx.x == 0) {
    s_timestep[slot] = timestep[i];
    s_action[slot] = action[i];
    s_reward[slot] = reward[i];
    s_nonterminal[slot] = nonterminal[i];
  }
}

// The window of sample d (redis_memory.py:347-369,479-541): ring slots idx-history+1 .. idx-history+L of the actor's
// segment, the blank frames across episode boundaries (:494-499) and the nonterminal flags after blanking (one thread).
__device__ __forceinline__ void window_slots(long d, int actor_cap, int history, int L,
                                             const int32_t* __restrict__ s_timestep,
                                             const uint8_t* __restrict__ s_nonterminal, long* slots, int* blank, int* nt) {
  const long actor = d / actor_cap;
  int ts[16];
  for (int k = 0; k < L; ++k) {
    long pos = (k + d - history + 1) % actor_cap;
    if (pos < 0) pos += actor_cap;
    slots[k] = pos + actor * actor_cap;
    ts[k] = s_timestep[slots[k]];
    nt[k] = s_nonterminal[slots[k]];
    blank[k] = 0;
  }
  for (int t = history - 2; t >= 0; --t)
    if (ts[t + 1] == 0) { blank[t] = 1; ts[t] = 0; nt[t] = 0; }
  for (int t = history; t < L; ++t)
    if (!nt[t - 1]) { blank[t] = 1; ts[t] = 0; nt[t] = 0; }
}

// The n-step return sum_k gamma^k r_{t+k} in float64, in the reference's order (:516-518).
__device__ __forceinline__ double n_step_return(int history, int n_step, const long* slots, const int* blank,
                                                const float* __restrict__ s_reward, const double* gamma_pow) {
  double ret = 0.0;
  for (int k = 0; k < n_step; ++k) {
    const int t = history + k - 1;
    const double r = blank[t] ? 0.0 : (double)s_reward[slots[t]];
    ret = __dadd_rn(ret, __dmul_rn(gamma_pow[k], r));   // python: sum(discount**k * reward), no FMA
  }
  return ret;
}

// Transition assembly (redis_memory.py:347-369,479-541): 7-frame window idx-3..idx+3 inside the actor's
// ring, blank frames across episode boundaries, n-step return in float64, output the uint8 window
// (B, history+n, 84, 84): states = window[:, :history], next_states = window[:, n:n+history].
__global__ void frame_gather_kernel(int B, int actor_cap, int history, int n_step, const int64_t* __restrict__ data_idx,
                                    const uint8_t* __restrict__ s_frames, const int32_t* __restrict__ s_timestep,
                                    const int32_t* __restrict__ s_action, const float* __restrict__ s_reward,
                                    const uint8_t* __restrict__ s_nonterminal, const double* __restrict__ gamma_pow,
                                    uint8_t* __restrict__ window, int64_t* __restrict__ actions,
                                    float* __restrict__ returns, float* __restrict__ nonterminals) {
  const int b = blockIdx.x;
  const int L = history + n_step;
  __shared__ long slots[16];
  __shared__ int blank[16];
  if (threadIdx.x == 0) {
    int nt[16];
    window_slots(data_idx[b], actor_cap, history, L, s_timestep, s_nonterminal, slots, blank, nt);
    returns[b] = (float)n_step_return(history, n_step, slots, blank, s_reward, gamma_pow);
    actions[b] = s_action[slots[history - 1]];
    nonterminals[b] = nt[L - 1] ? 1.f : 0.f;
  }
  __syncthreads();
  constexpr int V = FRAME_BYTES / 16;
  for (int t = threadIdx.x; t < L * V; t += blockDim.x) {
    const int k = t / V, o = t % V;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (!blank[k]) v = reinterpret_cast<const uint4*>(s_frames + slots[k] * FRAME_BYTES)[o];
    reinterpret_cast<uint4*>(window + ((long)b * L + k) * FRAME_BYTES)[o] = v;
  }
}

// frame_gather_kernel at this step's n = hz->n_step (kept in 1..n_max), read on the device, with a window of a fixed
// 2 * history frames: frames[:, :history] are the states and frames[:, history:] the next states (window frames
// n .. n+history-1), so their offsets do not depend on n.  discounts[b] = fl32(gamma^n) * nt_b.
__global__ void frame_gather_horizon_kernel(int B, int actor_cap, int history, int n_max,
                                            const int64_t* __restrict__ data_idx, const uint8_t* __restrict__ s_frames,
                                            const int32_t* __restrict__ s_timestep, const int32_t* __restrict__ s_action,
                                            const float* __restrict__ s_reward, const uint8_t* __restrict__ s_nonterminal,
                                            const riqn_horizon_state* __restrict__ hz, uint8_t* __restrict__ frames,
                                            int64_t* __restrict__ actions, float* __restrict__ returns,
                                            float* __restrict__ nonterminals, float* __restrict__ discounts) {
  const int b = blockIdx.x;
  const int n_step = min(max(hz->n_step, 1), n_max);
  const int L = history + n_step;
  __shared__ long slots[16];
  __shared__ int blank[16];
  if (threadIdx.x == 0) {
    int nt[16];
    window_slots(data_idx[b], actor_cap, history, L, s_timestep, s_nonterminal, slots, blank, nt);
    returns[b] = (float)n_step_return(history, n_step, slots, blank, s_reward, hz->gamma_pow);
    actions[b] = s_action[slots[history - 1]];
    const float ntf = nt[L - 1] ? 1.f : 0.f;
    nonterminals[b] = ntf;
    discounts[b] = __fmul_rn(hz->gamma_n, ntf);
  }
  __syncthreads();
  constexpr int V = FRAME_BYTES / 16;
  const int F = 2 * history;
  for (int t = threadIdx.x; t < F * V; t += blockDim.x) {
    const int k = t / V, o = t % V;
    const int w = k < history ? k : k - history + n_step;      // the window frame this output frame holds
    uint4 v = make_uint4(0, 0, 0, 0);
    if (!blank[w]) v = reinterpret_cast<const uint4*>(s_frames + slots[w] * FRAME_BYTES)[o];
    reinterpret_cast<uint4*>(frames + ((long)b * F + k) * FRAME_BYTES)[o] = v;
  }
}

// SPR's multi-step window: frame_gather_kernel's slots and blanking over history + K frames (no return), the K logged
// actions a_t .. a_{t+K-1}, and valid[b, k-1] for the step to s_{t+k}: its last frame is not blank and the walk
// p+1 .. p+k from the sampled ring position p does not reach the write head (past it lie older or unwritten slots).
__global__ void sequence_gather_kernel(int B, int actor_cap, int history, int K, const int64_t* __restrict__ data_idx,
                                       const int64_t* __restrict__ index_actor, const uint8_t* __restrict__ s_frames,
                                       const int32_t* __restrict__ s_timestep, const int32_t* __restrict__ s_action,
                                       const uint8_t* __restrict__ s_nonterminal, uint8_t* __restrict__ window,
                                       int64_t* __restrict__ actions, uint8_t* __restrict__ valid) {
  const int b = blockIdx.x;
  const int L = history + K;
  __shared__ long slots[16];
  __shared__ int blank[16];
  if (threadIdx.x == 0) {
    const long d = data_idx[b];
    const long actor = d / actor_cap;
    int nt[16];
    window_slots(d, actor_cap, history, L, s_timestep, s_nonterminal, slots, blank, nt);
    long head = (index_actor[actor] - d % actor_cap) % actor_cap;       // distance from p to the write head
    if (head < 0) head += actor_cap;
    for (int k = 0; k < K; ++k) {
      actions[(long)b * K + k] = s_action[slots[history - 1 + k]];
      valid[(long)b * K + k] = (!blank[history + k] && !(head >= 1 && head <= k + 1)) ? 1 : 0;
    }
  }
  __syncthreads();
  constexpr int V = FRAME_BYTES / 16;
  for (int t = threadIdx.x; t < L * V; t += blockDim.x) {
    const int k = t / V, o = t % V;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (!blank[k]) v = reinterpret_cast<const uint4*>(s_frames + slots[k] * FRAME_BYTES)[o];
    reinterpret_cast<uint4*>(window + ((long)b * L + k) * FRAME_BYTES)[o] = v;
  }
}

}  // namespace riqn

using namespace riqn;

RIQN_API int riqn_sumtree_stratified(int n, unsigned long long seed, unsigned long long stream_id, const double* tree,
                                     double* values, const riqn_dyn_state* dyn, void* stream) {
  riqn::note_launches(1);
  if (n <= 0 || n > 12000 || !tree || !values) return (int)cudaErrorInvalidValue;
  stratified_kernel<<<1, 1024, sizeof(int) * n, (cudaStream_t)stream>>>(n, seed, stream_id, tree, values, dyn);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_sumtree_sample(int n, long capacity, int actor_capacity, const double* tree, const double* values,
                                 const long long* index_actor, int history, int n_step, long long* tree_idx,
                                 long long* data_idx, double* priorities, void* stream) {
  riqn::note_launches(1);
  // the segment of a leaf is d / actor_capacity, so the segments must tile the tree exactly
  if (capacity < 1 || actor_capacity < 1 || capacity % actor_capacity != 0 || history < 0 || n_step < 0 || !tree ||
      !values || !index_actor || !tree_idx || !data_idx || !priorities)
    return (int)cudaErrorInvalidValue;
  if (n <= 0) return 0;
  const int warps_per_block = 4;
  sumtree_sample_kernel<false><<<riqn_cdiv(n, warps_per_block), warps_per_block * 32, 0, (cudaStream_t)stream>>>(
      n, capacity, actor_capacity, tree, values, (const int64_t*)index_actor, history, n_step, nullptr,
      (int64_t*)tree_idx, (int64_t*)data_idx, priorities);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_sumtree_sample_horizon(int n, long capacity, int actor_capacity, const double* tree,
                                         const double* values, const long long* index_actor, int history, int n_max,
                                         const riqn_horizon_state* hz, long long* tree_idx, long long* data_idx,
                                         double* priorities, void* stream) {
  riqn::note_launches(1);
  if (capacity < 1 || actor_capacity < 1 || capacity % actor_capacity != 0 || history < 0 || n_max < 1 ||
      n_max > RIQN_MAX_HORIZON || !tree || !values || !index_actor || !hz || !tree_idx || !data_idx || !priorities)
    return (int)cudaErrorInvalidValue;
  if (n <= 0) return 0;
  const int warps_per_block = 4;
  sumtree_sample_kernel<true><<<riqn_cdiv(n, warps_per_block), warps_per_block * 32, 0, (cudaStream_t)stream>>>(
      n, capacity, actor_capacity, tree, values, (const int64_t*)index_actor, history, n_max, hz, (int64_t*)tree_idx,
      (int64_t*)data_idx, priorities);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_sumtree_is_weights(int n, const double* tree, const double* priorities, double current_capacity,
                                     double priority_weight, double* w64, float* w32, int* n_nonpositive,
                                     const riqn_dyn_state* dyn, void* stream) {
  riqn::note_launches(1);
  if (n < 1 || !tree || !priorities || !w64 || !w32) return (int)cudaErrorInvalidValue;
  // with dyn the device values replace these (checked by whoever writes them).  A capacity of 0 (a tree filled without
  // the fill count) is accepted: like the reference's numpy, (0 * p)^-beta / max gives NaN weights
  if (!dyn && (!isfinite(current_capacity) || !(current_capacity >= 0.0) || !isfinite(priority_weight) ||
               !(priority_weight >= 0.0)))
    return (int)cudaErrorInvalidValue;
  is_weights_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(n, tree, priorities, current_capacity, priority_weight, w64,
                                                          w32, n_nonpositive, dyn);
  return (int)cudaGetLastError();
}

template <bool DEMO>
static int launch_sumtree_update(int n, long capacity, double* tree, const long long* tree_idx, const float* loss,
                                 float priority_exponent, int apply_pow, float* new_priorities, double* diff_scratch,
                                 double* max_priority, long long demo_leaf, float bonus, void* stream) {
  riqn::note_launches(2);
  if (capacity < 1 || !tree || !tree_idx || !loss || !new_priorities || !diff_scratch || !max_priority)
    return (int)cudaErrorInvalidValue;
  if (n <= 0) return 0;
  if (n > 4096) return (int)cudaErrorInvalidValue;  // shared-memory bound of the propagate kernel
  cudaStream_t s = (cudaStream_t)stream;
  update_prepare_kernel<DEMO><<<1, 1024, 0, s>>>(n, tree, (const int64_t*)tree_idx, loss, priority_exponent, apply_pow,
                                                 new_priorities, diff_scratch, max_priority, (int64_t)demo_leaf, bonus);
  RIQN_LAUNCH_CHECK();
  int max_depth = 0;  // depth of the deepest leaf (index 2C-2)
  for (long i = 2 * capacity - 2; i > 0; i = (i - 1) / 2) ++max_depth;
  const size_t smem = (size_t)n * 20;
  static PerDeviceOnce attr_once;
  const int attr_dev = PerDeviceOnce::device();
  if (!attr_once.done[attr_dev]) {
    RIQN_CUDA(cudaFuncSetAttribute(update_propagate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    attr_once.done[attr_dev] = true;
  }
  const int slices = (n + 63) / 64 < 8 ? (n + 63) / 64 : 8;      // 8 warps per CTA, one batch entry per warp at a time
  update_propagate_kernel<<<dim3(max_depth + 1, slices), 256, smem, s>>>(n, max_depth, tree, (const int64_t*)tree_idx,
                                                                        diff_scratch);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_sumtree_update(int n, long capacity, double* tree, const long long* tree_idx, const float* loss,
                                 float priority_exponent, int apply_pow, float* new_priorities, double* diff_scratch,
                                 double* max_priority, void* stream) {
  return launch_sumtree_update<false>(n, capacity, tree, tree_idx, loss, priority_exponent, apply_pow, new_priorities,
                                      diff_scratch, max_priority, 0, 0.f, stream);
}

RIQN_API int riqn_sumtree_update_demo(int n, long capacity, double* tree, const long long* tree_idx, const float* loss,
                                      float priority_exponent, int apply_pow, float* new_priorities, double* diff_scratch,
                                      double* max_priority, long long demo_leaf, float bonus, void* stream) {
  if (!(bonus >= 0.f) || !isfinite(bonus) || demo_leaf < 0) return (int)cudaErrorInvalidValue;
  return launch_sumtree_update<true>(n, capacity, tree, tree_idx, loss, priority_exponent, apply_pow, new_priorities,
                                     diff_scratch, max_priority, demo_leaf, bonus, stream);
}

RIQN_API int riqn_replay_append(int n, int actor_capacity, int id_actor, int start, const unsigned char* frames,
                                const int* timestep, const int* action, const float* reward,
                                const unsigned char* nonterminal, unsigned char* s_frames, int* s_timestep, int* s_action,
                                float* s_reward, unsigned char* s_nonterminal, void* stream) {
  riqn::note_launches(1);
  // n <= actor_capacity: one launch writes every slot at most once (more would let two blocks race on a slot)
  if (actor_capacity < 1 || id_actor < 0 || start < 0 || start >= actor_capacity || n > actor_capacity || !frames ||
      !timestep || !action || !reward || !nonterminal || !s_frames || !s_timestep || !s_action || !s_reward ||
      !s_nonterminal)
    return (int)cudaErrorInvalidValue;
  if (n <= 0) return 0;
  replay_append_kernel<<<n, 128, 0, (cudaStream_t)stream>>>(n, actor_capacity, id_actor, start, frames, timestep, action,
                                                            reward, nonterminal, s_frames, s_timestep, s_action, s_reward,
                                                            s_nonterminal);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_frame_gather(int batch, int actor_capacity, int history, int n_step, const long long* data_idx,
                               const unsigned char* s_frames, const int* s_timestep, const int* s_action,
                               const float* s_reward, const unsigned char* s_nonterminal, const double* gamma_pow,
                               unsigned char* window, long long* actions, float* returns, float* nonterminals,
                               void* stream) {
  riqn::note_launches(1);
  if (actor_capacity < 1 || history < 1 || n_step < 1 || history + n_step > 16 || !data_idx || !s_frames ||
      !s_timestep || !s_action || !s_reward || !s_nonterminal || !gamma_pow || !window || !actions || !returns ||
      !nonterminals)
    return (int)cudaErrorInvalidValue;
  if (batch <= 0) return 0;
  frame_gather_kernel<<<batch, 256, 0, (cudaStream_t)stream>>>(batch, actor_capacity, history, n_step,
                                                               (const int64_t*)data_idx, s_frames, s_timestep, s_action,
                                                               s_reward, s_nonterminal, gamma_pow, window,
                                                               (int64_t*)actions, returns, nonterminals);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_frame_gather_horizon(int batch, int actor_capacity, int history, int n_max, const long long* data_idx,
                                       const unsigned char* s_frames, const int* s_timestep, const int* s_action,
                                       const float* s_reward, const unsigned char* s_nonterminal,
                                       const riqn_horizon_state* hz, unsigned char* frames, long long* actions,
                                       float* returns, float* nonterminals, float* discounts, void* stream) {
  riqn::note_launches(1);
  if (actor_capacity < 1 || history < 1 || n_max < 1 || history + n_max > 16 || !data_idx || !s_frames ||
      !s_timestep || !s_action || !s_reward || !s_nonterminal || !hz || !frames || !actions || !returns ||
      !nonterminals || !discounts)
    return (int)cudaErrorInvalidValue;
  if (batch <= 0) return 0;
  frame_gather_horizon_kernel<<<batch, 256, 0, (cudaStream_t)stream>>>(
      batch, actor_capacity, history, n_max, (const int64_t*)data_idx, s_frames, s_timestep, s_action, s_reward,
      s_nonterminal, hz, frames, (int64_t*)actions, returns, nonterminals, discounts);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_sequence_gather(int batch, int actor_capacity, int history, int K, const long long* data_idx,
                                  const long long* index_actor, const unsigned char* s_frames, const int* s_timestep,
                                  const int* s_action, const unsigned char* s_nonterminal, unsigned char* window,
                                  long long* actions, unsigned char* valid, void* stream) {
  if (batch < 1 || actor_capacity < 1 || history < 1 || K < 1 || history + K > 16 || !data_idx || !index_actor ||
      !s_frames || !s_timestep || !s_action || !s_nonterminal || !window || !actions || !valid)
    return (int)cudaErrorInvalidValue;
  riqn::note_launches(1);
  sequence_gather_kernel<<<batch, 256, 0, (cudaStream_t)stream>>>(
      batch, actor_capacity, history, K, (const int64_t*)data_idx, (const int64_t*)index_actor, s_frames, s_timestep,
      s_action, s_nonterminal, window, (int64_t*)actions, valid);
  return (int)cudaGetLastError();
}
