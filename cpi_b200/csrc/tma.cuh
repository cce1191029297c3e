// 1-D TMA bulk copy + mbarrier primitives shared by the preintegration kernels (SASS: UBLKCP / SYNCS).
#pragma once
#include "cpi_common.cuh"

namespace cpi {

// ---- TMA (1-D bulk copy) + mbarrier primitives: SASS UBLKCP / SYNCS ---------------------------------------------------
CPI_DEV uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
CPI_DEV void mbar_init(uint32_t bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory"); }
CPI_DEV void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
CPI_DEV void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}
CPI_DEV void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    } while (!ok);
}
CPI_DEV void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

CPI_DEV void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
// before an mbarrier's memory is reused for anything else
CPI_DEV void mbar_inval(uint32_t bar) { asm volatile("mbarrier.inval.shared::cta.b64 [%0];" ::"r"(bar) : "memory"); }

}  // namespace cpi
