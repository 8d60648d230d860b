// ABI version + device check entry points.
#include "common.cuh"
#include "../../include/heal_b200.h"

extern "C" int heal_abi_version(void) { return HEAL_B200_ABI_VERSION; }

extern "C" int heal_device_check(void) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return HEAL_ERR_DRIVER;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) return HEAL_ERR_DRIVER;
    return (prop.major == 9) ? HEAL_OK : HEAL_ERR_UNSUPPORTED;
}

#include <atomic>
static std::atomic<long long> g_heal_launches{0};
extern "C" void heal_launch_counter_add(int n) { g_heal_launches.fetch_add(n, std::memory_order_relaxed); }
extern "C" long long heal_launch_count(void) { return g_heal_launches.load(std::memory_order_relaxed); }
