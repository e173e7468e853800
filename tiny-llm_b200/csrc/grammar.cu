// Grammar-constrained generation (DESIGN.md section 23): the token masks and the state advance of a table-driven
// byte-level pushdown automaton compiled from a GBNF grammar, walked over a *set* of live parses (the blob layout and
// the row state are in include/tiny_llm_b200.h, written and mirrored bit for bit by tiny_llm_b200/grammar.py).
//
// Masks: one CTA row per batch row, one thread per token.  The CTA stages its row's live parse set (the parses' states,
// depths and return stacks) and byte classes in shared memory, and its table blob too when it fits the launch's
// dynamic shared memory (sized by the caller to the largest blob that fits, as for the schema kernel).  A thread walks
// its token's bytes over up to TL_GRAMMAR_MAX_PARSES parses held in local memory: a parse keeps the entries it pushed
// in a private overlay above its base, and entries below the base are read from its staged row stack, so forking a
// parse copies only what this token pushed.  After every byte the new parses are deduplicated by (state, depth, stack)
// as they are made; one more distinct parse than the cap refuses the token.  A warp covers 32 consecutive tokens and
// writes the mask word with one ballot.  No atomics: every launch writes the same words.
//
// Advance: one thread per row, after the draw, walks the drawn token for rows with position > 0 and writes the new
// parse set, or sets the failed bit when the token was not allowed (only past the parse cap).
#include "common.cuh"
#include "kernels.h"

namespace tl {

namespace {

constexpr int GRAMMAR_THREADS = 256;
constexpr int WORDS = TL_GRAMMAR_STATE_WORDS;
constexpr int MAX_DEPTH = TL_GRAMMAR_MAX_DEPTH;
constexpr int MAX_PARSES = TL_GRAMMAR_MAX_PARSES;
constexpr int STACK_WORD = 2 + MAX_PARSES;  // the first int64 word of the return stacks
constexpr uint32_t INFO_MAY_END = 1u;
constexpr uint64_t ACTIVE = 1ull << 32, TERMINAL = 1ull << 33, FAILED = 1ull << 34;
constexpr int HEADER_BYTES = 16 + 256;  // four int32 and class_of
static_assert(WORDS == STACK_WORD + MAX_PARSES * MAX_DEPTH / 4, "the row state holds every parse's stack");
static_assert(TL_GRAMMAR_SMEM_BYTES + 2 * MAX_PARSES * MAX_DEPTH + 256 + 4 * MAX_PARSES + 4 <= 48 * 1024,
              "the staged blob, row stacks, parse heads and byte classes fit the default shared memory");

struct Tables {
    const uint8_t *class_of;  // always the CTA's shared copy in the masks kernel
    const uint32_t *info;
    const uint32_t *trans;
    const uint32_t *acts;
    uint32_t classes;

    __device__ __forceinline__ void bind(const uint8_t *base) {
        const int32_t *h = reinterpret_cast<const int32_t *>(base);
        const int S = h[0];
        classes = static_cast<uint32_t>(h[1]);
        class_of = base + 16;
        info = reinterpret_cast<const uint32_t *>(base + HEADER_BYTES);
        trans = info + S;
        acts = trans + static_cast<size_t>(S) * classes;
    }
};

// One parse of a token walk: entries below base are the row's stack of parse src, entries from base up to depth are
// the overlay.
struct Parse {
    uint16_t s, depth, base, src;
    uint16_t overlay[MAX_DEPTH];
};

__device__ __forceinline__ uint32_t entry_of(const Parse &p, const uint16_t *stacks, int k) {
    return k < p.base ? stacks[p.src * MAX_DEPTH + k] : p.overlay[k];
}

__device__ __forceinline__ uint32_t pushed(const uint32_t *rets, uint32_t x) { return (rets[x >> 1] >> (16 * (x & 1))) & 0xFFFFu; }

__device__ __forceinline__ uint32_t pop(Parse &p, const uint16_t *stacks) {
    const int d = --p.depth;
    if (d >= p.base) return p.overlay[d];
    p.base = static_cast<uint16_t>(d);
    return stacks[p.src * MAX_DEPTH + d];
}

// One byte over the parses cur[0, n) into nxt: every action of each parse's state on the byte's class, then (while the
// state's rule may end and the stack is not empty) the same after popping the return state.  Returns the new count,
// or -1 past the parse cap.  cur's parses are consumed.
__device__ __forceinline__ int step_set(const Tables &t, const uint16_t *stacks, Parse *cur, int n, Parse *nxt, uint32_t b) {
    const uint32_t c = t.class_of[b];
    int m = 0;
    for (int i = 0; i < n; ++i) {
        Parse &w = cur[i];
        while (true) {
            const uint32_t e = t.trans[w.s * t.classes + c];
            uint32_t off = e & 0xFFFFFFu;
            const uint32_t count = e >> 24;
            for (uint32_t a = 0; a < count; ++a) {
                const uint32_t word = t.acts[off];
                const uint32_t target = word & 0x7FFFu, k = (word >> 16) & 63u, peak = word >> 24;
                const uint32_t *rets = t.acts + off + 1;
                off += 1 + ((k + 1) >> 1);
                if (w.depth + peak > MAX_DEPTH) continue;
                const int depth = w.depth + k;
                bool dup = false;
                for (int j = 0; j < m && !dup; ++j) {
                    const Parse &q = nxt[j];
                    if (q.s != target || q.depth != depth) continue;
                    bool same = true;
                    for (int x = depth - 1; x >= 0 && same; --x) {
                        if (x < w.base && x < q.base && w.src == q.src) break;  // both read the same row stack below
                        const uint32_t va = x >= w.depth ? pushed(rets, x - w.depth) : entry_of(w, stacks, x);
                        same = va == entry_of(q, stacks, x);
                    }
                    dup = same;
                }
                if (dup) continue;
                if (m == MAX_PARSES) return -1;
                Parse &q = nxt[m++];
                q.s = static_cast<uint16_t>(target);
                q.depth = static_cast<uint16_t>(depth);
                q.base = w.base;
                q.src = w.src;
                for (int x = w.base; x < w.depth; ++x) q.overlay[x] = w.overlay[x];
                for (uint32_t x = 0; x < k; ++x) q.overlay[w.depth + x] = static_cast<uint16_t>(pushed(rets, x));
            }
            if (!(t.info[w.s] & INFO_MAY_END) || w.depth == 0) break;
            w.s = static_cast<uint16_t>(pop(w, stacks));
        }
    }
    return m;
}

// Some parse has finished root at depth 0, returning through states whose rule may end.
__device__ __forceinline__ bool complete(const Tables &t, const uint16_t *stacks, const uint32_t *heads, int n) {
    for (int p = 0; p < n; ++p) {
        uint32_t s = heads[p] & 0x7FFFu, d = (heads[p] >> 16) & 63u;
        while (t.info[s] & INFO_MAY_END) {
            if (d == 0) return true;
            s = stacks[p * MAX_DEPTH + --d];
        }
    }
    return false;
}

__device__ __forceinline__ void load_set(Parse *cur, const uint32_t *heads, int n) {
    for (int p = 0; p < n; ++p) {
        cur[p].s = static_cast<uint16_t>(heads[p] & 0x7FFFu);
        cur[p].depth = cur[p].base = static_cast<uint16_t>((heads[p] >> 16) & 63u);
        cur[p].src = static_cast<uint16_t>(p);
    }
}

__global__ void __launch_bounds__(GRAMMAR_THREADS)
    grammar_masks_kernel(const tl_constraint_row *__restrict__ con, const int64_t *__restrict__ states, int vocab) {
    extern __shared__ uint4 staged_blob[];
    __shared__ uint16_t stacks[MAX_PARSES * MAX_DEPTH];
    __shared__ uint32_t class_of[64];
    __shared__ uint32_t heads[MAX_PARSES];
    __shared__ int row_complete;
    const int row = blockIdx.y;
    const int64_t *st = states + static_cast<size_t>(row) * WORDS;
    const uint64_t w1 = static_cast<uint64_t>(st[1]);
    if (!(w1 & ACTIVE) || (w1 & TERMINAL)) return;  // not a grammar row, or after EOS: the EOS-only row applies
    const uint8_t *blob = reinterpret_cast<const uint8_t *>(st[0]);
    const int nbytes = __ldg(reinterpret_cast<const int32_t *>(blob) + 2);
    uint32_t dynamic_smem;
    asm("mov.u32 %0, %%dynamic_smem_size;" : "=r"(dynamic_smem));
    const bool staged = static_cast<uint32_t>(nbytes) <= dynamic_smem;
    if (staged) {
        const uint4 *src = reinterpret_cast<const uint4 *>(blob);
        for (int i = threadIdx.x; i < (nbytes >> 4); i += GRAMMAR_THREADS) staged_blob[i] = __ldg(src + i);
    }
    if (threadIdx.x < MAX_PARSES * MAX_DEPTH / 2)
        reinterpret_cast<uint32_t *>(stacks)[threadIdx.x] = reinterpret_cast<const uint32_t *>(st + STACK_WORD)[threadIdx.x];
    if (threadIdx.x < MAX_PARSES) heads[threadIdx.x] = static_cast<uint32_t>(st[2 + threadIdx.x]);
    if (threadIdx.x < 64) class_of[threadIdx.x] = __ldg(reinterpret_cast<const uint32_t *>(blob + 16) + threadIdx.x);
    __syncthreads();
    Tables tab;
    tab.bind(staged ? reinterpret_cast<const uint8_t *>(staged_blob) : blob);
    tab.class_of = reinterpret_cast<const uint8_t *>(class_of);
    const int n = static_cast<int>(w1 & 15u);
    if (threadIdx.x == 0) row_complete = complete(tab, stacks, heads, n);
    __syncthreads();

    const int32_t *offsets = con[row].token_offsets;
    const uint8_t *bytes = con[row].token_bytes;
    const int W = (vocab + 31) >> 5;
    uint32_t *mask = const_cast<uint32_t *>(con[row].mask);
    const int t = blockIdx.x * GRAMMAR_THREADS + threadIdx.x;
    const int word = t >> 5;  // the same for the 32 lanes of a warp
    if (word >= W) return;    // whole warps only
    bool ok = false;
    if (t < vocab) {
        const int b0 = __ldg(offsets + t), b1 = __ldg(offsets + t + 1);
        if (b1 > b0) {
            Parse buf[2][MAX_PARSES];
            Parse *cur = buf[0], *nxt = buf[1];
            load_set(cur, heads, n);
            int m = n;
            for (int j = b0; j < b1 && m > 0; ++j) {
                m = step_set(tab, stacks, cur, m, nxt, __ldg(bytes + j));
                Parse *tmp = cur;
                cur = nxt;
                nxt = tmp;
            }
            ok = m > 0;
        } else {
            ok = row_complete && ((__ldg(mask + W + word) >> (t & 31)) & 1u);
        }
    }
    const unsigned bits = __ballot_sync(0xffffffffu, ok);
    if ((threadIdx.x & 31) == 0) mask[word] = bits;
}

__global__ void grammar_advance_kernel(const tl_constraint_row *__restrict__ con, int64_t *__restrict__ states,
                                       const int32_t *__restrict__ tokens, const int32_t *__restrict__ positions, int rows, int vocab) {
    const int row = blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= rows) return;
    int64_t *st = states + static_cast<size_t>(row) * WORDS;
    const uint64_t w1 = static_cast<uint64_t>(st[1]);
    if (!(w1 & ACTIVE) || (w1 & (TERMINAL | FAILED)) || positions[row] <= 0) return;
    Tables tab;
    tab.bind(reinterpret_cast<const uint8_t *>(st[0]));
    uint16_t stacks[MAX_PARSES * MAX_DEPTH];
    uint32_t heads[MAX_PARSES];
    const uint16_t *src = reinterpret_cast<const uint16_t *>(st + STACK_WORD);
    for (int k = 0; k < MAX_PARSES * MAX_DEPTH; ++k) stacks[k] = src[k];
    for (int p = 0; p < MAX_PARSES; ++p) heads[p] = static_cast<uint32_t>(st[2 + p]);
    const int n = static_cast<int>(w1 & 15u);
    const int token = tokens[row];
    const int b0 = con[row].token_offsets[token], b1 = con[row].token_offsets[token + 1];
    if (b0 == b1) {  // no bytes: EOS ends a complete text; any other id was not allowed
        const int W = (vocab + 31) >> 5;
        const bool eos = (con[row].mask[W + (token >> 5)] >> (token & 31)) & 1u;
        if (eos && complete(tab, stacks, heads, n)) {
            st[1] = static_cast<int64_t>(w1 | TERMINAL);
            return;
        }
    }
    Parse buf[2][MAX_PARSES];
    Parse *cur = buf[0], *nxt = buf[1];
    load_set(cur, heads, n);
    int m = b0 == b1 ? 0 : n;
    for (int j = b0; j < b1 && m > 0; ++j) {
        m = step_set(tab, stacks, cur, m, nxt, con[row].token_bytes[j]);
        Parse *tmp = cur;
        cur = nxt;
        nxt = tmp;
    }
    const bool failed = m <= 0;  // a token outside the language or past the parse cap (drawn only when none is allowed)
    if (failed) m = 0;
    uint64_t packed[MAX_PARSES * MAX_DEPTH / 4] = {};
    for (int p = 0; p < MAX_PARSES; ++p) {
        st[2 + p] = p < m ? static_cast<int64_t>(cur[p].s | (static_cast<uint32_t>(cur[p].depth) << 16)) : 0;
        if (p >= m) continue;
        for (int k = 0; k < cur[p].depth; ++k) {
            const int at = p * MAX_DEPTH + k;
            packed[at >> 2] |= static_cast<uint64_t>(entry_of(cur[p], stacks, k)) << (16 * (at & 3));
        }
    }
    for (int k = 0; k < MAX_PARSES * MAX_DEPTH / 4; ++k) st[STACK_WORD + k] = static_cast<int64_t>(packed[k]);
    st[1] = static_cast<int64_t>((w1 & ~15ull) | static_cast<uint64_t>(m) | (failed ? FAILED : 0));
}

}  // namespace

int launch_grammar_token_masks(const tl_constraint_row *constraints, const int64_t *states, int rows, int vocab, int smem_bytes,
                               cudaStream_t st) {
    if (rows == 0) return TL_OK;
    grammar_masks_kernel<<<dim3(ceil_div(vocab, GRAMMAR_THREADS), rows), GRAMMAR_THREADS, smem_bytes, st>>>(constraints, states, vocab);
    TL_LAUNCH_CHECK("grammar_token_masks");
    return TL_OK;
}

int launch_grammar_advance(const tl_constraint_row *constraints, int64_t *states, const int32_t *tokens, const int32_t *positions, int rows,
                           int vocab, cudaStream_t st) {
    if (rows == 0) return TL_OK;
    grammar_advance_kernel<<<ceil_div(rows, 64), 64, 0, st>>>(constraints, states, tokens, positions, rows, vocab);
    TL_LAUNCH_CHECK("grammar_advance");
    return TL_OK;
}

}  // namespace tl
