// Tensor maps (TMA descriptors) for the wgmma kernels: the swap-AB W4A16 GEMM (w4a16_skinny.cu) and the paged
// FlashAttention kernel (attention_prefill_tc.cu).
#include <array>
#include <mutex>
#include <unordered_map>

#include "common.cuh"
#include "wgmma.cuh"

namespace tl {

// cuTensorMapEncodeTiled through the runtime (no link-time dependency on libcuda).
static PFN_cuTensorMapEncodeTiled_v12000 tensor_map_encoder() {
    static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
    }
    return fn;
}

namespace {
constexpr int MAX_RANK = 4;

struct MapKey {
    const void *ptr;
    CUtensorMapDataType dtype;
    int rank;
    std::array<cuuint64_t, MAX_RANK> dims;
    std::array<cuuint32_t, MAX_RANK> box;
    CUtensorMapSwizzle swizzle;
    CUtensorMapL2promotion l2;
    bool operator==(const MapKey &o) const {
        return ptr == o.ptr && dtype == o.dtype && rank == o.rank && dims == o.dims && box == o.box && swizzle == o.swizzle && l2 == o.l2;
    }
};
struct MapKeyHash {
    size_t operator()(const MapKey &k) const {
        size_t h = reinterpret_cast<size_t>(k.ptr);
        auto mix = [&h](unsigned long long v) { h = h * 1000003u ^ static_cast<size_t>(v); };
        mix(k.dtype), mix(k.rank), mix(k.swizzle), mix(k.l2);
        for (int i = 0; i < k.rank; ++i) mix(k.dims[i]), mix(k.box[i]);
        return h;
    }
};
}  // namespace

// Cached per operand: a model re-uses a handful of distinct operands (weights, activation and K/V buffers) in every
// layer and step, and cuTensorMapEncodeTiled costs microseconds per call.
int cached_tensor_map(CUtensorMap *out, const void *ptr, CUtensorMapDataType dtype, int rank, const cuuint64_t *dims, const cuuint32_t *box,
                      CUtensorMapSwizzle swizzle, CUtensorMapL2promotion l2, const char *what) {
    if (rank < 1 || rank > MAX_RANK) return fail(TL_EINVAL, "%s: tensor map of rank %d", what, rank);
    static std::mutex mu;
    static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
    MapKey key{ptr, dtype, rank, {}, {}, swizzle, l2};
    for (int i = 0; i < rank; ++i) key.dims[i] = dims[i], key.box[i] = box[i];
    std::lock_guard<std::mutex> lock(mu);
    auto it = cache.find(key);
    if (it != cache.end()) {
        *out = it->second;
        return TL_OK;
    }
    PFN_cuTensorMapEncodeTiled_v12000 encode = tensor_map_encoder();
    if (encode == nullptr) return fail(TL_ECUDA, "%s: cuTensorMapEncodeTiled is unavailable", what);
    // Dense row-major tensors of bytes (packed weights) or 16-bit floats: the stride of dimension i + 1 is the byte size
    // of everything below it.
    cuuint64_t strides[MAX_RANK - 1];
    cuuint64_t acc = dtype == CU_TENSOR_MAP_DATA_TYPE_UINT8 ? 1 : 2;
    for (int i = 0; i + 1 < rank; ++i) {
        acc *= dims[i];
        strides[i] = acc;
    }
    const cuuint32_t estr[MAX_RANK] = {1, 1, 1, 1};
    CUtensorMap map;
    CUresult r = encode(&map, dtype, rank, const_cast<void *>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, l2,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(TL_ECUDA, "%s: cuTensorMapEncodeTiled failed (%d)", what, static_cast<int>(r));
    if (cache.size() > 8192) cache.clear();
    cache.emplace(key, map);
    *out = map;
    return TL_OK;
}

}  // namespace tl
