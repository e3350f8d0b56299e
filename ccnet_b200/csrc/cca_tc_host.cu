// Host-side helpers of the wgmma kernels: tensor-map cache, per-device SM count.
#include <mutex>
#include <unordered_map>

#include "cca_tc_common.cuh"

namespace cca {
namespace tc {
namespace {
struct MapKey {
    const void *base;
    int B, H, W, C, LK, flags;
    bool operator==(const MapKey &o) const
    {
        return base == o.base && B == o.B && H == o.H && W == o.W && C == o.C && LK == o.LK && flags == o.flags;
    }
};
struct MapKeyHash {
    size_t operator()(const MapKey &k) const
    {
        size_t h = reinterpret_cast<size_t>(k.base);
        auto mix = [&](size_t v) { h ^= v + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2); };
        mix((size_t)k.B); mix((size_t)k.H); mix((size_t)k.W); mix((size_t)k.C); mix((size_t)k.LK); mix((size_t)k.flags);
        return h;
    }
};
std::mutex g_map_mu;
std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_maps;
constexpr size_t kMaxCachedMaps = 1024;

std::mutex g_sm_mu;
int g_sm_count[64] = {};
}  // namespace

bool get_map(CUtensorMap *m, const void *base, int B, int H, int W, int C, int LK, bool col, bool bf16)
{
    int dev = 0;
    cudaGetDevice(&dev);                       // the same virtual address may be a different tensor on another device
    const MapKey key{base, B, H, W, C, LK, (col ? 1 : 0) | (bf16 ? 2 : 0) | (dev << 2)};
    {
        std::lock_guard<std::mutex> lk(g_map_mu);
        auto it = g_maps.find(key);
        if (it != g_maps.end()) { *m = it->second; return true; }
    }
    if (!make_map(m, base, B, H, W, C, LK, col, bf16)) return false;
    std::lock_guard<std::mutex> lk(g_map_mu);
    if (g_maps.size() >= kMaxCachedMaps) g_maps.clear();
    g_maps.emplace(key, *m);
    return true;
}

int sm_count()
{
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
    std::lock_guard<std::mutex> lk(g_sm_mu);
    if (!g_sm_count[dev]) cudaDeviceGetAttribute(&g_sm_count[dev], cudaDevAttrMultiProcessorCount, dev);
    return g_sm_count[dev] > 0 ? g_sm_count[dev] : 132;
}

}  // namespace tc
}  // namespace cca
