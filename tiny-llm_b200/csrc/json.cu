// JSON mode (DESIGN.md section 20): the token masks and the state advance of a byte-level pushdown automaton whose
// state is kept per row on the device, two int64 words (the layout is in include/tiny_llm_b200.h and mirrored by
// tiny_llm_b200/json_mode.py, which must agree bit for bit).
//
// Masks: one CTA row per batch row, one thread per token.  The thread walks the token's bytes from the row's state in
// registers, with its own copy of the container stack word; a warp covers 32 consecutive tokens and writes the mask
// word with one ballot.  A token without bytes is allowed exactly when the text is complete and the row's EOS-only
// mask (row 1 of its buffer) has its bit.  No atomics: every launch writes the same words.
//
// Advance: one thread per row, after the draw, walks the drawn token for rows with position > 0 (idle slots and
// capture warm-ups change nothing), as tl_sample_constrained gates its own state advance.
#include "common.cuh"
#include "kernels.h"

namespace tl {

namespace {

constexpr int JSON_THREADS = 256;

// Lexer states (bits 8-12 of word 1).
enum : uint32_t {
    J_START = 0,      // before the top-level '{'
    J_OBJ_FIRST = 1,  // after '{': '"' or '}'
    J_OBJ_KEY = 2,    // after ',' in an object: '"'
    J_COLON = 3,      // after a key: ':'
    J_VALUE = 4,      // after ':' or ',' in an array: a value
    J_ARR_FIRST = 5,  // after '[': a value or ']'
    J_AFTER = 6,      // after a value in a container: ',' or the matching close
    J_CLOSED = 7,     // after the top-level '}': whitespace, then EOS
    J_STR = 8,        // in a string
    J_ESC = 9,        // after '\'
    J_HEX = 10,       // in \uXXXX, aux hex digits to go
    J_UTF8 = 11,      // in a multi-byte character, aux continuation bytes to go, aux2 the next byte's range
    J_MINUS = 12,
    J_ZERO = 13,
    J_INT = 14,
    J_DOT = 15,
    J_FRAC = 16,
    J_EXP_MARK = 17,
    J_EXP_SIGN = 18,
    J_EXP = 19,
    J_LIT = 20,  // in true / false / null: aux the literal, aux2 the next byte's index
    J_DEAD = 31,
};

constexpr uint32_t DEPTH_MASK = 0x7Fu;
constexpr int LEX_SHIFT = 8, WS_SHIFT = 16, AUX_SHIFT = 24, AUX2_SHIFT = 27, KEY_BIT = 30;
constexpr uint64_t ACTIVE = 1ull << 32, TERMINAL = 1ull << 33;

__device__ __forceinline__ bool is_ws(uint32_t b) { return b == 0x20 || b == 0x09 || b == 0x0A || b == 0x0D; }
__device__ __forceinline__ bool is_digit(uint32_t b) { return b - '0' < 10u; }

// Byte k of literal `lit` (0 true, 1 false, 2 null) and its length.
__device__ __forceinline__ uint32_t lit_byte(uint32_t lit, uint32_t k) {
    const uint64_t w = lit == 0 ? 0x65757274ull : lit == 1 ? 0x65736c6166ull : 0x6c6c756eull;  // little-endian bytes
    return static_cast<uint32_t>(w >> (8 * k)) & 0xFFu;
}
__device__ __forceinline__ uint32_t lit_len(uint32_t lit) { return lit == 1 ? 5u : 4u; }

struct Pda {
    uint64_t stack;  // bit d: the container at depth d + 1 is an array
    uint32_t depth, lex, ws, aux, aux2, key;

    __device__ __forceinline__ void load(uint64_t w0, uint64_t w1) {
        const uint32_t s = static_cast<uint32_t>(w1);
        stack = w0;
        depth = s & DEPTH_MASK;
        lex = (s >> LEX_SHIFT) & 31u;
        ws = (s >> WS_SHIFT) & 63u;
        aux = (s >> AUX_SHIFT) & 7u;
        aux2 = (s >> AUX2_SHIFT) & 7u;
        key = (s >> KEY_BIT) & 1u;
    }
    __device__ __forceinline__ uint32_t word() const {
        return depth | (lex << LEX_SHIFT) | (ws << WS_SHIFT) | (aux << AUX_SHIFT) | (aux2 << AUX2_SHIFT) | (key << KEY_BIT);
    }
    __device__ __forceinline__ bool top_array() const { return (stack >> (depth - 1)) & 1ull; }

    __device__ __forceinline__ bool push(bool array) {
        if (depth >= JSON_MAX_DEPTH_) return false;
        stack = array ? (stack | (1ull << depth)) : (stack & ~(1ull << depth));
        ++depth;
        lex = array ? J_ARR_FIRST : J_OBJ_FIRST;
        return true;
    }
    __device__ __forceinline__ void pop() {
        --depth;
        lex = depth == 0 ? J_CLOSED : J_AFTER;
    }
    static constexpr uint32_t JSON_MAX_DEPTH_ = TL_JSON_MAX_DEPTH;

    // A value's first byte (in J_VALUE or J_ARR_FIRST).
    __device__ __forceinline__ bool value_start(uint32_t b) {
        if (b == '{') return push(false);
        if (b == '[') return push(true);
        if (b == '"') return lex = J_STR, key = 0, true;
        if (b == '-') return lex = J_MINUS, true;
        if (b == '0') return lex = J_ZERO, true;
        if (is_digit(b)) return lex = J_INT, true;
        if (b == 't' || b == 'f' || b == 'n') return lex = J_LIT, aux = b == 't' ? 0 : b == 'f' ? 1 : 2, aux2 = 1, true;
        return false;
    }
    // A byte after a complete value inside a container.
    __device__ __forceinline__ bool after_value(uint32_t b) {
        lex = J_AFTER;
        if (b == ',') return lex = top_array() ? J_VALUE : J_OBJ_KEY, true;
        if (b == (top_array() ? ']' : '}')) return pop(), true;
        return false;
    }

    // One byte; false when it leaves the language (the state is then unspecified).
    __device__ __forceinline__ bool step(uint32_t b) {
        const bool number_may_end = lex == J_ZERO || lex == J_INT || lex == J_FRAC || lex == J_EXP;
        if (lex <= J_CLOSED || number_may_end) {  // whitespace counts here; elsewhere the run is already 0
            if (is_ws(b)) {
                if (number_may_end) lex = J_AFTER;
                if (ws >= TL_JSON_MAX_WS_RUN) return false;
                ++ws;
                return true;
            }
            ws = 0;
        }
        switch (lex) {
            case J_START:
                return b == '{' && push(false);
            case J_OBJ_FIRST:
                if (b == '}') return pop(), true;
                return b == '"' && (lex = J_STR, key = 1, true);
            case J_OBJ_KEY:
                return b == '"' && (lex = J_STR, key = 1, true);
            case J_COLON:
                return b == ':' && (lex = J_VALUE, true);
            case J_VALUE:
                return value_start(b);
            case J_ARR_FIRST:
                if (b == ']') return pop(), true;
                return value_start(b);
            case J_AFTER:
                return after_value(b);
            case J_CLOSED:
                return false;
            case J_STR:
                if (b == '"') return lex = key ? J_COLON : J_AFTER, key = 0, true;
                if (b == '\\') return lex = J_ESC, true;
                if (b >= 0x20 && b < 0x80) return true;
                if (b >= 0xC2 && b <= 0xDF) return lex = J_UTF8, aux = 1, aux2 = 0, true;
                if (b >= 0xE0 && b <= 0xEF) return lex = J_UTF8, aux = 2, aux2 = b == 0xE0 ? 1 : b == 0xED ? 2 : 0, true;
                if (b >= 0xF0 && b <= 0xF4) return lex = J_UTF8, aux = 3, aux2 = b == 0xF0 ? 3 : b == 0xF4 ? 4 : 0, true;
                return false;
            case J_ESC:
                if (b == 'u') return lex = J_HEX, aux = 4, true;
                return (b == '"' || b == '\\' || b == '/' || b == 'b' || b == 'f' || b == 'n' || b == 'r' || b == 't') && (lex = J_STR, true);
            case J_HEX:
                if (!(is_digit(b) || (b | 0x20u) - 'a' < 6u)) return false;
                if (--aux == 0) lex = J_STR;
                return true;
            case J_UTF8: {
                // next-byte ranges: 0 80-BF, 1 A0-BF (after E0), 2 80-9F (after ED), 3 90-BF (after F0), 4 80-8F (after F4)
                const uint32_t lo = aux2 == 1 ? 0xA0 : aux2 == 3 ? 0x90 : 0x80;
                const uint32_t hi = aux2 == 2 ? 0x9F : aux2 == 4 ? 0x8F : 0xBF;
                if (b < lo || b > hi) return false;
                aux2 = 0;
                if (--aux == 0) lex = J_STR;
                return true;
            }
            case J_MINUS:
                if (b == '0') return lex = J_ZERO, true;
                return is_digit(b) && (lex = J_INT, true);
            case J_ZERO:
                if (b == '.') return lex = J_DOT, true;
                if ((b | 0x20u) == 'e') return lex = J_EXP_MARK, true;
                return after_value(b);
            case J_INT:
                if (is_digit(b)) return true;
                if (b == '.') return lex = J_DOT, true;
                if ((b | 0x20u) == 'e') return lex = J_EXP_MARK, true;
                return after_value(b);
            case J_DOT:
                return is_digit(b) && (lex = J_FRAC, true);
            case J_FRAC:
                if (is_digit(b)) return true;
                if ((b | 0x20u) == 'e') return lex = J_EXP_MARK, true;
                return after_value(b);
            case J_EXP_MARK:
                if (b == '+' || b == '-') return lex = J_EXP_SIGN, true;
                return is_digit(b) && (lex = J_EXP, true);
            case J_EXP_SIGN:
                return is_digit(b) && (lex = J_EXP, true);
            case J_EXP:
                if (is_digit(b)) return true;
                return after_value(b);
            case J_LIT:
                if (b != lit_byte(aux, aux2)) return false;
                if (++aux2 == lit_len(aux)) lex = J_AFTER, aux = 0, aux2 = 0;
                return true;
            default:
                return false;
        }
    }
};

__global__ void __launch_bounds__(JSON_THREADS)
    json_masks_kernel(const tl_constraint_row *__restrict__ con, const int64_t *__restrict__ states, int vocab) {
    const int row = blockIdx.y;
    const uint64_t w1 = static_cast<uint64_t>(states[2 * row + 1]);
    if (!(w1 & ACTIVE) || (w1 & TERMINAL)) return;  // not a JSON row, or after EOS: the EOS-only row applies
    const uint64_t w0 = static_cast<uint64_t>(states[2 * row]);
    const int32_t *offsets = con[row].token_offsets;
    const uint8_t *bytes = con[row].token_bytes;
    const int W = (vocab + 31) >> 5;
    uint32_t *mask = const_cast<uint32_t *>(con[row].mask);
    const int t = blockIdx.x * JSON_THREADS + threadIdx.x;
    const int word = t >> 5;  // the same for the 32 lanes of a warp
    if (word >= W) return;    // whole warps only
    Pda start;
    start.load(w0, w1);
    bool ok = false;
    if (t < vocab) {
        const int b0 = __ldg(offsets + t), b1 = __ldg(offsets + t + 1);
        if (b1 > b0) {
            Pda p = start;
            ok = p.lex != J_DEAD;
            for (int j = b0; j < b1 && ok; ++j) ok = p.step(__ldg(bytes + j));
        } else {
            ok = start.lex == J_CLOSED && ((__ldg(mask + W + word) >> (t & 31)) & 1u);
        }
    }
    const unsigned bits = __ballot_sync(0xffffffffu, ok);
    if ((threadIdx.x & 31) == 0) mask[word] = bits;
}

__global__ void json_advance_kernel(const tl_constraint_row *__restrict__ con, int64_t *__restrict__ states, const int32_t *__restrict__ tokens,
                                    const int32_t *__restrict__ positions, int rows) {
    const int row = blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= rows) return;
    uint64_t w1 = static_cast<uint64_t>(states[2 * row + 1]);
    if (!(w1 & ACTIVE) || (w1 & TERMINAL) || positions[row] <= 0) return;
    const int token = tokens[row];
    const int b0 = con[row].token_offsets[token], b1 = con[row].token_offsets[token + 1];
    if (b0 == b1) {  // EOS (the only allowed token without bytes)
        states[2 * row + 1] = static_cast<int64_t>(w1 | TERMINAL);
        return;
    }
    Pda p;
    p.load(static_cast<uint64_t>(states[2 * row]), w1);
    bool ok = p.lex != J_DEAD;
    for (int j = b0; j < b1 && ok; ++j) ok = p.step(con[row].token_bytes[j]);
    if (!ok) p = Pda{p.stack, p.depth, J_DEAD, 0, 0, 0, 0};  // a token outside the language (never drawn): nothing is allowed after it
    states[2 * row] = static_cast<int64_t>(p.stack);
    states[2 * row + 1] = static_cast<int64_t>((w1 & ~0xFFFFFFFFull) | p.word());
}

}  // namespace

int launch_json_token_masks(const tl_constraint_row *constraints, const int64_t *states, int rows, int vocab, cudaStream_t st) {
    if (rows == 0) return TL_OK;
    json_masks_kernel<<<dim3(ceil_div(vocab, JSON_THREADS), rows), JSON_THREADS, 0, st>>>(constraints, states, vocab);
    TL_LAUNCH_CHECK("json_token_masks");
    return TL_OK;
}

int launch_json_advance(const tl_constraint_row *constraints, int64_t *states, const int32_t *tokens, const int32_t *positions, int rows,
                        cudaStream_t st) {
    if (rows == 0) return TL_OK;
    json_advance_kernel<<<ceil_div(rows, 64), 64, 0, st>>>(constraints, states, tokens, positions, rows);
    TL_LAUNCH_CHECK("json_advance");
    return TL_OK;
}

}  // namespace tl
