// JSON Schema structured outputs (DESIGN.md section 21): the token masks and the state advance of a table-driven
// byte-level pushdown automaton compiled from a schema (the blob layout and the row state are in
// include/tiny_llm_b200.h, written and mirrored bit for bit by tiny_llm_b200/json_schema.py).
//
// Masks: one CTA row per batch row, one thread per token.  The CTA stages its row's table blob in shared memory when it
// fits the launch's dynamic shared memory (the caller sizes it to the largest blob of its rows, at most
// TL_SCHEMA_SMEM_BYTES, so a launch whose rows fit none keeps its occupancy), and its byte classes and stack of return
// states always; a row whose blob does not fit reads it through L1/L2 with the same result.  A thread walks its token's bytes from the row's state in registers; the stack entries it
// pushes go to a private overlay, and entries below the row's top are read from the staged row stack.  A warp covers 32
// consecutive tokens and writes the mask word with one ballot.  No atomics: every launch writes the same words.
//
// Advance: one thread per row, after the draw, walks the drawn token for rows with position > 0, as tl_json_advance.
#include "common.cuh"
#include "kernels.h"

namespace tl {

namespace {

constexpr int SCHEMA_THREADS = 256;
constexpr int WORDS = TL_SCHEMA_STATE_WORDS;
constexpr int MAX_DEPTH = TL_SCHEMA_MAX_DEPTH;
constexpr uint32_t K_CHECKED_SHIFT = 0, K_CALL = 1, K_RETURN = 2, K_REPROCESS = 3, K_SHIFT = 4, K_FAIL = 5;
constexpr uint32_t INFO_WS = 1u, INFO_ACCEPT = 2u;
constexpr uint64_t ACTIVE = 1ull << 32, TERMINAL = 1ull << 33;
constexpr int HEADER_BYTES = 16 + 256;  // four int32 and class_of
static_assert(TL_SCHEMA_SMEM_BYTES + 2 * MAX_DEPTH + 256 <= 48 * 1024, "the staged blob, row stack and byte classes fit the default shared memory");

__device__ __forceinline__ bool is_ws(uint32_t b) { return b == 0x20 || b == 0x09 || b == 0x0A || b == 0x0D; }
__device__ __forceinline__ uint32_t need_of(uint32_t info) { return (info >> 8) & 0xFFu; }

struct Tables {
    const uint8_t *class_of;  // always the CTA's shared copy in the masks kernel
    const uint32_t *info;
    const uint32_t *actions;
    const uint16_t *trans;
    uint32_t classes;

    __device__ __forceinline__ void bind(const uint8_t *base) {
        const int32_t *h = reinterpret_cast<const int32_t *>(base);
        const int S = h[0], A = h[3];
        classes = static_cast<uint32_t>(h[1]);
        class_of = base + 16;
        info = reinterpret_cast<const uint32_t *>(base + HEADER_BYTES);
        actions = info + S;
        trans = reinterpret_cast<const uint16_t *>(actions + A);
    }
    // (kind, target, return) of state s on byte class c; a plain shift needs no depth check
    __device__ __forceinline__ uint32_t entry(uint32_t s, uint32_t c, uint32_t &target, uint32_t &ret) const {
        const uint32_t e = trans[s * classes + c];
        if (!(e & 0x8000u)) return target = e, e ? K_SHIFT : K_FAIL;
        const uint32_t a = actions[e & 0x7FFFu];
        target = (a >> 2) & 0x7FFFu;
        ret = (a >> 17) & 0x7FFFu;
        return a & 3u;
    }
};

struct Walk {
    uint32_t s, depth, ws, base;  // base: the row stack's entries below it are still the row's
    uint16_t overlay[MAX_DEPTH];  // entries this walk pushed, at their stack positions

    __device__ __forceinline__ void load(uint64_t w1) {
        s = static_cast<uint32_t>(w1) & 0x7FFFu;
        depth = (static_cast<uint32_t>(w1) >> 16) & 63u;
        ws = (static_cast<uint32_t>(w1) >> 24) & 63u;
        base = depth;
    }
    __device__ __forceinline__ uint32_t pop(const uint16_t *row_stack) {
        --depth;
        if (depth >= base) return overlay[depth];
        base = depth;
        return row_stack[depth];
    }

    // One byte; false when it leaves the language (the state is then unspecified).
    __device__ __forceinline__ bool step(const Tables &t, const uint16_t *row_stack, uint32_t b) {
        const uint32_t c = t.class_of[b];
        uint32_t target = 0, ret = 0;
        uint32_t kind = t.entry(s, c, target, ret);
        if (kind == K_REPROCESS) {  // a number ended: the byte belongs to the caller's return state
            if (depth == 0) return false;
            s = pop(row_stack);
            kind = t.entry(s, c, target, ret);
            if (kind == K_REPROCESS) return false;
        }
        if (kind == K_FAIL) return false;
        // the run is nonzero only in whitespace states, so a byte that is not whitespace resets it anywhere
        if (!is_ws(b)) {
            ws = 0;
        } else if (t.info[s] & INFO_WS) {
            if (ws >= TL_JSON_MAX_WS_RUN) return false;
            ++ws;
        }
        if (kind == K_SHIFT) {
            s = target;
            return true;
        }
        if (kind == K_CHECKED_SHIFT) {
            if (depth + need_of(t.info[target]) > MAX_DEPTH) return false;
            s = target;
            return true;
        }
        if (kind == K_CALL) {
            if (depth + 1 + need_of(t.info[target]) > MAX_DEPTH || depth + need_of(t.info[ret]) > MAX_DEPTH) return false;
            overlay[depth++] = static_cast<uint16_t>(ret);
            s = target;
            return true;
        }
        if (kind != K_RETURN || depth == 0) return false;
        s = pop(row_stack);
        return true;
    }
};

__global__ void __launch_bounds__(SCHEMA_THREADS)
    schema_masks_kernel(const tl_constraint_row *__restrict__ con, const int64_t *__restrict__ states, int vocab) {
    extern __shared__ uint4 staged_blob[];
    __shared__ uint16_t row_stack[MAX_DEPTH];
    __shared__ uint32_t class_of[64];
    const int row = blockIdx.y;
    const int64_t *st = states + static_cast<size_t>(row) * WORDS;
    const uint64_t w1 = static_cast<uint64_t>(st[1]);
    if (!(w1 & ACTIVE) || (w1 & TERMINAL)) return;  // not a schema row, or after EOS: the EOS-only row applies
    const uint8_t *blob = reinterpret_cast<const uint8_t *>(st[0]);
    const int nbytes = __ldg(reinterpret_cast<const int32_t *>(blob) + 2);
    uint32_t dynamic_smem;
    asm("mov.u32 %0, %%dynamic_smem_size;" : "=r"(dynamic_smem));
    const bool staged = static_cast<uint32_t>(nbytes) <= dynamic_smem;
    if (staged) {
        const uint4 *src = reinterpret_cast<const uint4 *>(blob);
        for (int i = threadIdx.x; i < (nbytes >> 4); i += SCHEMA_THREADS) staged_blob[i] = __ldg(src + i);
    }
    if (threadIdx.x < MAX_DEPTH) row_stack[threadIdx.x] = reinterpret_cast<const uint16_t *>(st + 2)[threadIdx.x];
    if (threadIdx.x < 64) class_of[threadIdx.x] = __ldg(reinterpret_cast<const uint32_t *>(blob + 16) + threadIdx.x);
    __syncthreads();
    Tables tab;
    tab.bind(staged ? reinterpret_cast<const uint8_t *>(staged_blob) : blob);
    tab.class_of = reinterpret_cast<const uint8_t *>(class_of);

    const int32_t *offsets = con[row].token_offsets;
    const uint8_t *bytes = con[row].token_bytes;
    const int W = (vocab + 31) >> 5;
    uint32_t *mask = const_cast<uint32_t *>(con[row].mask);
    const int t = blockIdx.x * SCHEMA_THREADS + threadIdx.x;
    const int word = t >> 5;  // the same for the 32 lanes of a warp
    if (word >= W) return;    // whole warps only
    Walk w;
    w.load(w1);
    bool ok = false;
    if (t < vocab) {
        const int b0 = __ldg(offsets + t), b1 = __ldg(offsets + t + 1);
        if (b1 > b0) {
            ok = w.s != 0;
            for (int j = b0; j < b1 && ok; ++j) ok = w.step(tab, row_stack, __ldg(bytes + j));
        } else {
            ok = (tab.info[w.s] & INFO_ACCEPT) && w.depth == 0 && ((__ldg(mask + W + word) >> (t & 31)) & 1u);
        }
    }
    const unsigned bits = __ballot_sync(0xffffffffu, ok);
    if ((threadIdx.x & 31) == 0) mask[word] = bits;
}

__global__ void schema_advance_kernel(const tl_constraint_row *__restrict__ con, int64_t *__restrict__ states,
                                      const int32_t *__restrict__ tokens, const int32_t *__restrict__ positions, int rows) {
    const int row = blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= rows) return;
    int64_t *st = states + static_cast<size_t>(row) * WORDS;
    const uint64_t w1 = static_cast<uint64_t>(st[1]);
    if (!(w1 & ACTIVE) || (w1 & TERMINAL) || positions[row] <= 0) return;
    const int token = tokens[row];
    const int b0 = con[row].token_offsets[token], b1 = con[row].token_offsets[token + 1];
    if (b0 == b1) {  // EOS (the only allowed token without bytes)
        st[1] = static_cast<int64_t>(w1 | TERMINAL);
        return;
    }
    Tables tab;
    tab.bind(reinterpret_cast<const uint8_t *>(st[0]));
    uint16_t row_stack[MAX_DEPTH];
    const uint16_t *src = reinterpret_cast<const uint16_t *>(st + 2);
    for (int k = 0; k < MAX_DEPTH; ++k) row_stack[k] = src[k];
    Walk w;
    w.load(w1);
    bool ok = w.s != 0;
    for (int j = b0; j < b1 && ok; ++j) ok = w.step(tab, row_stack, con[row].token_bytes[j]);
    if (!ok) w.s = w.depth = w.ws = w.base = 0;  // a token outside the language (never drawn): the dead state
    uint64_t packed[(MAX_DEPTH + 3) / 4] = {};
    for (uint32_t k = 0; k < w.depth; ++k) packed[k >> 2] |= static_cast<uint64_t>(k < w.base ? row_stack[k] : w.overlay[k]) << (16 * (k & 3));
    for (int k = 0; k < (MAX_DEPTH + 3) / 4; ++k) st[2 + k] = static_cast<int64_t>(packed[k]);
    st[1] = static_cast<int64_t>((w1 & ~0xFFFFFFFFull) | w.s | (w.depth << 16) | (w.ws << 24));
}

}  // namespace

int launch_schema_token_masks(const tl_constraint_row *constraints, const int64_t *states, int rows, int vocab, int smem_bytes,
                              cudaStream_t st) {
    if (rows == 0) return TL_OK;
    schema_masks_kernel<<<dim3(ceil_div(vocab, SCHEMA_THREADS), rows), SCHEMA_THREADS, smem_bytes, st>>>(constraints, states, vocab);
    TL_LAUNCH_CHECK("schema_token_masks");
    return TL_OK;
}

int launch_schema_advance(const tl_constraint_row *constraints, int64_t *states, const int32_t *tokens, const int32_t *positions, int rows,
                          cudaStream_t st) {
    if (rows == 0) return TL_OK;
    schema_advance_kernel<<<ceil_div(rows, 64), 64, 0, st>>>(constraints, states, tokens, positions, rows);
    TL_LAUNCH_CHECK("schema_advance");
    return TL_OK;
}

}  // namespace tl
