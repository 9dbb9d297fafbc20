// seal_b200/csrc/sb_api.cu -- the extern "C" boundary declared in include/seal_b200.h.
// Exceptions never cross it: they are mapped to status codes the way the reference's C layer maps them to HRESULTs
// (native/src/seal/c/defines.h:72-96) and the message is kept in a thread-local string.  The evaluator operations, the CKKS
// encoder and the decryptor are each described once (what they check, their slab layout, their launch on a chunk of the batch)
// and get their stream and host-buffer entry points from the two drivers on_stream and on_host.
#include "../../include/seal_b200.h"
#include "sb_engine.cuh"
#include <random>
#include <algorithm>
#include <array>
#include <cctype>
#include <cstdio>
#include <cstring>
#include <new>
#include <thread>

using namespace sb;

static thread_local std::string g_last_error;

struct sb200_context
{
    std::unique_ptr<Context> c;
};
// the key's device memory is freed (the secret key's wiped first) by its members, on the context's device
struct sb200_public_key
{
    PublicKey k;
    ~sb200_public_key()
    {
        if (k.ctx)
            cudaSetDevice(k.ctx->device);
    }
};
struct sb200_secret_key
{
    SecretKey k;
    ~sb200_secret_key()
    {
        if (k.ctx)
            cudaSetDevice(k.ctx->device);
    }
};
struct sb200_kswitch_key
{
    KSwitchKey k;
    ~sb200_kswitch_key()
    {
        if (k.ctx)
            cudaSetDevice(k.ctx->device);
    }
};

// a missing pointer found inside SB_TRY: SB200_E_POINTER, as SB_NEED returns
struct null_pointer : std::runtime_error
{
    explicit null_pointer(const std::string &what) : std::runtime_error("null pointer: " + what) {}
};

#define SB_TRY try {
#define SB_CATCH                                   \
    }                                              \
    catch (const null_pointer &e)                  \
    {                                              \
        g_last_error = e.what();                   \
        return SB200_E_POINTER;                    \
    }                                              \
    catch (const std::invalid_argument &e)         \
    {                                              \
        g_last_error = e.what();                   \
        return SB200_E_INVALID_ARG;                \
    }                                              \
    catch (const std::out_of_range &e)             \
    {                                              \
        g_last_error = e.what();                   \
        return SB200_E_OUT_OF_RANGE;               \
    }                                              \
    catch (const std::logic_error &e)              \
    {                                              \
        g_last_error = e.what();                   \
        return SB200_E_LOGIC;                      \
    }                                              \
    catch (const std::bad_alloc &e)                \
    {                                              \
        g_last_error = e.what();                   \
        return SB200_E_NOMEM;                      \
    }                                              \
    catch (const std::exception &e)                \
    {                                              \
        g_last_error = e.what();                   \
        return SB200_E_CUDA;                       \
    }

#define SB_NEED(p)                                      \
    if (!(p))                                           \
    {                                                   \
        g_last_error = "null pointer: " #p;             \
        return SB200_E_POINTER;                         \
    }

extern "C" {

const char *sb200_last_error(void)
{
    return g_last_error.c_str();
}

int sb200_context_create(int scheme, size_t n, const uint64_t *coeff_modulus, size_t k, uint64_t plain_modulus, int device,
                         sb200_context **out)
{
    SB_NEED(coeff_modulus);
    SB_NEED(out);
    SB_TRY
    auto h = std::make_unique<sb200_context>();
    h->c = make_context(scheme, n, reinterpret_cast<const u64 *>(coeff_modulus), k, plain_modulus, device);
    *out = h.release();
    return SB200_OK;
    SB_CATCH
}

int sb200_context_destroy(sb200_context *ctx)
{
    SB_NEED(ctx);
    delete ctx;
    return SB200_OK;
}

int sb200_coeff_modulus_create(size_t n, const int *bit_sizes, size_t k, uint64_t *out)
{
    SB_NEED(bit_sizes);
    SB_NEED(out);
    SB_TRY
    if (n < 2 || (n & (n - 1)) || n > 131072)
        throw std::invalid_argument("poly_modulus_degree is invalid");
    for (size_t i = 0; i < k; i++)
        if (bit_sizes[i] < 2 || bit_sizes[i] > 60)
            throw std::invalid_argument("bit_sizes is invalid");
    auto v = sbh::coeff_modulus_create(n, std::vector<int>(bit_sizes, bit_sizes + k));
    for (size_t i = 0; i < k; i++)
        out[i] = v[i];
    return SB200_OK;
    SB_CATCH
}

int sb200_get_ntt_tables(const sb200_context *ctx, size_t i, uint64_t *root, uint64_t *rp_op, uint64_t *rp_quo, uint64_t *irp_op,
                         uint64_t *inv_n)
{
    SB_NEED(ctx);
    SB_TRY
    const Context &c = *ctx->c;
    if (i >= c.k)
        throw std::out_of_range("prime_index");
    const auto &t = c.tabs[i];
    if (root)
        *root = t.root;
    if (inv_n)
        *inv_n = t.inv_n.w;
    for (size_t j = 0; j < c.n; j++)
    {
        if (rp_op)
            rp_op[j] = t.root_powers[j].w;
        if (rp_quo)
            rp_quo[j] = t.root_powers[j].wq;
        if (irp_op)
            irp_op[j] = t.inv_root_powers[j].w;
    }
    return SB200_OK;
    SB_CATCH
}

int sb200_get_base_bsk(const sb200_context *ctx, size_t L, uint64_t *out, size_t capacity, size_t *count)
{
    SB_NEED(ctx);
    SB_NEED(out);
    SB_NEED(count);
    SB_TRY
    Context &c = *ctx->c;
    if (c.scheme != SB200_SCHEME_BFV)
        throw std::logic_error("BEHZ base exists for BFV contexts only");
    const auto &b = behz_host(c, L);
    if (b.nBsk > capacity)
        throw std::out_of_range("capacity");
    for (size_t i = 0; i < b.nBsk; i++)
        out[i] = b.Bsk[i];
    *count = b.nBsk;
    return SB200_OK;
    SB_CATCH
}

uint32_t sb200_galois_elt_from_step(const sb200_context *ctx, int step)
{
    if (!ctx)
        return 0;
    try
    {
        return sbh::galois_elt_from_step(ctx->c->n, step);
    }
    catch (const std::exception &e)
    {
        g_last_error = e.what();
        return 0;
    }
}

unsigned long long sb200_launch_count(const sb200_context *ctx)
{
    return ctx ? ctx->c->stats.launches : 0;
}

size_t sb200_device_bytes(const sb200_context *ctx)
{
    return ctx ? ctx->c->table_bytes + ctx->c->scratch.bytes() + ctx->c->aux_buf.bytes() : 0;
}

int sb200_context_set_limit(sb200_context *ctx, int which, size_t value)
{
    SB_NEED(ctx);
    SB_TRY
    Context &c = *ctx->c;
    std::lock_guard<std::mutex> lock(c.mu);
    switch (which)
    {
    case SB200_LIMIT_SCRATCH_BYTES: c.scratch_budget = std::max<size_t>(value, size_t(1) << 20); break;
    case SB200_LIMIT_KS_CHUNK: c.ks_chunk_max = value; break;
    case SB200_LIMIT_HOST_STAGE_BYTES: c.host_stage_bytes = std::max<size_t>(value, size_t(1) << 16); break;
    case SB200_LIMIT_KS_ALGORITHM:
        if (value > 2)
            throw std::invalid_argument("unknown key-switching algorithm");
        c.ks_algo = static_cast<int>(value);
        break;
    default: throw std::invalid_argument("unknown limit");
    }
    return SB200_OK;
    SB_CATCH
}

// ---- device-resident slabs / staging memory ----
int sb200_device_malloc(sb200_context *ctx, size_t bytes, uint64_t **d_out)
{
    SB_NEED(ctx);
    SB_NEED(d_out);
    SB_TRY
    Context &c = *ctx->c;
    cuda_check(cudaSetDevice(c.device), "cudaSetDevice");
    void *p = nullptr;
    cudaError_t e = cudaMalloc(&p, std::max<size_t>(bytes, 8));
    if (e == cudaErrorMemoryAllocation)
    {
        cudaGetLastError();
        throw std::bad_alloc();
    }
    cuda_check(e, "cudaMalloc(slab)");
    *d_out = static_cast<uint64_t *>(p);
    return SB200_OK;
    SB_CATCH
}
int sb200_device_free(sb200_context *ctx, uint64_t *d_ptr)
{
    SB_NEED(ctx);
    SB_TRY
    cuda_check(cudaSetDevice(ctx->c->device), "cudaSetDevice");
    cuda_check(cudaFree(d_ptr), "cudaFree(slab)");
    return SB200_OK;
    SB_CATCH
}
int sb200_host_malloc(sb200_context *ctx, size_t bytes, void **h_out)
{
    SB_NEED(ctx);
    SB_NEED(h_out);
    SB_TRY
    cuda_check(cudaSetDevice(ctx->c->device), "cudaSetDevice");
    void *p = nullptr;
    cudaError_t e = cudaHostAlloc(&p, std::max<size_t>(bytes, 8), cudaHostAllocDefault);
    if (e == cudaErrorMemoryAllocation)
    {
        cudaGetLastError();
        throw std::bad_alloc();
    }
    cuda_check(e, "cudaHostAlloc");
    *h_out = p;
    return SB200_OK;
    SB_CATCH
}
int sb200_host_free(sb200_context *ctx, void *h_ptr)
{
    SB_NEED(ctx);
    SB_TRY
    cuda_check(cudaFreeHost(h_ptr), "cudaFreeHost");
    return SB200_OK;
    SB_CATCH
}
static int copy_(sb200_context *ctx, void *dst, const void *src, size_t bytes, cudaMemcpyKind kind, void *stream)
{
    SB_NEED(ctx);
    SB_NEED(dst);
    SB_NEED(src);
    SB_TRY
    cuda_check(cudaSetDevice(ctx->c->device), "cudaSetDevice");
    cuda_check(cudaMemcpyAsync(dst, src, bytes, kind, static_cast<cudaStream_t>(stream)), "cudaMemcpyAsync");
    return SB200_OK;
    SB_CATCH
}
int sb200_memcpy_h2d(sb200_context *ctx, uint64_t *d_dst, const void *h_src, size_t bytes, void *stream)
{
    return copy_(ctx, d_dst, h_src, bytes, cudaMemcpyHostToDevice, stream);
}
int sb200_memcpy_d2h(sb200_context *ctx, void *h_dst, const uint64_t *d_src, size_t bytes, void *stream)
{
    return copy_(ctx, h_dst, d_src, bytes, cudaMemcpyDeviceToHost, stream);
}
int sb200_memcpy_d2d(sb200_context *ctx, uint64_t *d_dst, const uint64_t *d_src, size_t bytes, void *stream)
{
    return copy_(ctx, d_dst, d_src, bytes, cudaMemcpyDeviceToDevice, stream);
}
int sb200_memcpy_d2d_2d(sb200_context *ctx, uint64_t *d_dst, size_t dst_pitch, const uint64_t *d_src, size_t src_pitch, size_t row_bytes,
                        size_t rows, void *stream)
{
    SB_NEED(ctx);
    SB_NEED(d_dst);
    SB_NEED(d_src);
    SB_TRY
    cuda_check(cudaSetDevice(ctx->c->device), "cudaSetDevice");
    cuda_check(cudaMemcpy2DAsync(d_dst, dst_pitch, d_src, src_pitch, row_bytes, rows, cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream)),
               "cudaMemcpy2DAsync");
    return SB200_OK;
    SB_CATCH
}
int sb200_stream_synchronize(sb200_context *ctx, void *stream)
{
    SB_NEED(ctx);
    SB_TRY
    cuda_check(cudaSetDevice(ctx->c->device), "cudaSetDevice");
    cuda_check(cudaStreamSynchronize(static_cast<cudaStream_t>(stream)), "cudaStreamSynchronize");
    return SB200_OK;
    SB_CATCH
}
} // extern "C"
namespace
{
    // copies rows [r0, r1) between the caller's objects and a contiguous page-locked buffer on a few host threads (one thread
    // moves ~10 GB/s, a Gen5 x16 link 50+ GB/s)
    void rows_copy(bool gather, uint8_t *stage, const uint64_t *const *rows, size_t row_bytes, size_t r0, size_t r1)
    {
        const size_t cnt = r1 - r0;
        const unsigned hw = std::max(1u, std::thread::hardware_concurrency());
        const size_t nt = std::max<size_t>(1, std::min<size_t>({ 8, hw / 2 ? hw / 2 : 1, cnt * row_bytes / (size_t(4) << 20) + 1 }));
        auto work = [&](size_t t) {
            // split by bytes so that few large rows still spread over all threads
            const size_t total = cnt * row_bytes, b0 = total * t / nt, b1 = total * (t + 1) / nt;
            for (size_t off = b0; off < b1;)
            {
                const size_t r = off / row_bytes, in = off % row_bytes, len = std::min(row_bytes - in, b1 - off);
                uint8_t *user = reinterpret_cast<uint8_t *>(const_cast<uint64_t *>(rows[r0 + r])) + in;
                if (gather)
                    std::memcpy(stage + off, user, len);
                else
                    std::memcpy(user, stage + off, len);
                off += len;
            }
        };
        if (nt == 1)
            return work(0);
        std::vector<std::thread> th;
        for (size_t t = 1; t < nt; t++)
            th.emplace_back(work, t);
        work(0);
        for (auto &x : th)
            x.join();
    }
    void ensure_lane(IoArena::Lane &ln, size_t bytes)
    {
        if (!ln.st)
            ln.st = make_stream();
        for (auto *e : { &ln.order, &ln.ev[0], &ln.ev[1] })
            if (!*e)
                *e = make_event();
        for (auto &p : ln.pin)
            p.grow(bytes);
    }
    // The copies run on the lane's own non-blocking stream: they overlap kernels of other batches.  Ordering with the caller's
    // work: a download first waits for everything the legacy default stream has been given so far (the batch operations of the
    // C++ shim enqueue there); an upload returns when the data has arrived, so whatever the caller enqueues next sees it.
    // dev_pitch: bytes from one device row to the next (0: rows are contiguous); after_default = false: the caller has already
    // synchronised the work that wrote the rows, so the download does not wait for the legacy default stream
    void rows_transfer(Context &c, bool upload, uint64_t *dev, const uint64_t *const *rows, size_t row_bytes, size_t count, size_t dev_pitch = 0,
                       bool after_default = true)
    {
        if (!dev_pitch)
            dev_pitch = row_bytes;
        if (!count || !row_bytes)
            return;
        IoArena::Lane &ln = c.io.lane[upload ? 0 : 1];
        std::lock_guard<std::mutex> lock(ln.mu);
        cuda_check(cudaSetDevice(c.device), "cudaSetDevice");
        const size_t per = std::max<size_t>(1, (size_t(128) << 20) / row_bytes), stage_bytes = std::min(per, count) * row_bytes;
        ensure_lane(ln, stage_bytes);
        cudaStream_t st = ln.st.get();
        if (!upload && after_default)
        {
            cuda_check(cudaEventRecord(ln.order.get(), nullptr), "record");
            cuda_check(cudaStreamWaitEvent(st, ln.order.get(), 0), "wait");
        }
        uint8_t *d = reinterpret_cast<uint8_t *>(dev);
        size_t i = 0, pend[2] = { 0, 0 }, pend_n[2] = { 0, 0 };
        bool used[2] = { false, false };
        for (size_t r0 = 0; r0 < count; r0 += per, i++)
        {
            const size_t r1 = std::min(count, r0 + per);
            const int slot = static_cast<int>(i & 1);
            uint8_t *stage = ln.pin[slot].get();
            if (used[slot])
            {
                cuda_check(cudaEventSynchronize(ln.ev[slot].get()), "cudaEventSynchronize");
                if (!upload)
                    rows_copy(false, stage, rows, row_bytes, pend[slot], pend[slot] + pend_n[slot]);
            }
            if (upload)
            {
                rows_copy(true, stage, rows, row_bytes, r0, r1);
                cuda_check(cudaMemcpyAsync(d + r0 * row_bytes, stage, (r1 - r0) * row_bytes, cudaMemcpyHostToDevice, st), "H2D");
            }
            else if (dev_pitch == row_bytes)
                cuda_check(cudaMemcpyAsync(stage, d + r0 * row_bytes, (r1 - r0) * row_bytes, cudaMemcpyDeviceToHost, st), "D2H");
            else
                cuda_check(cudaMemcpy2DAsync(stage, row_bytes, d + r0 * dev_pitch, dev_pitch, row_bytes, r1 - r0, cudaMemcpyDeviceToHost, st),
                           "D2H");
            cuda_check(cudaEventRecord(ln.ev[slot].get(), st), "record");
            used[slot] = true, pend[slot] = r0, pend_n[slot] = r1 - r0;
        }
        // drain in submission order
        for (size_t j = (i >= 2 ? i - 2 : 0); j < i; j++)
        {
            const int slot = static_cast<int>(j & 1);
            cuda_check(cudaEventSynchronize(ln.ev[slot].get()), "cudaEventSynchronize");
            if (!upload)
                rows_copy(false, ln.pin[slot].get(), rows, row_bytes, pend[slot], pend[slot] + pend_n[slot]);
        }
    }
} // namespace
extern "C" {
int sb200_upload_rows(sb200_context *ctx, uint64_t *d_dst, const uint64_t *const *h_rows, size_t row_bytes, size_t count)
{
    SB_NEED(d_dst);
    SB_NEED(h_rows);
    SB_TRY
    SB_NEED(ctx);
    rows_transfer(*ctx->c, true, d_dst, h_rows, row_bytes, count);
    return SB200_OK;
    SB_CATCH
}
int sb200_download_rows(sb200_context *ctx, uint64_t *const *h_rows, const uint64_t *d_src, size_t row_bytes, size_t count)
{
    SB_NEED(d_src);
    SB_NEED(h_rows);
    SB_TRY
    SB_NEED(ctx);
    rows_transfer(*ctx->c, false, const_cast<uint64_t *>(d_src), h_rows, row_bytes, count);
    return SB200_OK;
    SB_CATCH
}
int sb200_device_index(const sb200_context *ctx)
{
    return ctx ? ctx->c->device : -1;
}
int sb200_device_numa_node(const sb200_context *ctx)
{
    if (!ctx)
        return -1;
    char bus[32] = { 0 };
    if (cudaDeviceGetPCIBusId(bus, sizeof(bus), ctx->c->device) != cudaSuccess)
        return -1;
    for (char *p = bus; *p; p++)
        *p = static_cast<char>(std::tolower(*p));
    std::string path = std::string("/sys/bus/pci/devices/") + bus + "/numa_node";
    int node = -1;
    if (FILE *f = std::fopen(path.c_str(), "r"))
    {
        if (std::fscanf(f, "%d", &node) != 1)
            node = -1;
        std::fclose(f);
    }
    return node;
}
size_t sb200_keyswitch_chunk(const sb200_context *ctx, size_t L, size_t batch, int fused)
{
    return ctx ? sb::keyswitch_chunk(*ctx->c, L, batch, fused != 0) : 0;
}

int sb200_profile_enable(sb200_context *ctx, int on)
{
    SB_NEED(ctx);
    std::lock_guard<std::mutex> lock(ctx->c->mu);
    ctx->c->stats.profiling = (on != 0);
    return SB200_OK;
}

int sb200_profile_reset(sb200_context *ctx)
{
    SB_NEED(ctx);
    std::lock_guard<std::mutex> lock(ctx->c->mu);
    cudaSetDevice(ctx->c->device);
    cudaDeviceSynchronize();
    ctx->c->stats.clear();
    return SB200_OK;
}

int sb200_profile_read(sb200_context *ctx, size_t index, char *name, size_t name_capacity, double *total_ms,
                       unsigned long long *launches, double *algorithmic_bytes)
{
    return sb200_profile_read_work(ctx, index, name, name_capacity, total_ms, launches, algorithmic_bytes, nullptr, nullptr);
}

int sb200_selftest_ksint_info(sb200_context *ctx, int *count, uint32_t *primes)
{
    SB_NEED(ctx);
    SB_NEED(count);
    SB_NEED(primes);
    const KsInt &d = ctx->c->ksint;
    *count = d.ready ? d.prm.S : 0;
    for (int t = 0; t < *count; t++)
        primes[t] = d.prm.p[t];
    return SB200_OK;
}

int sb200_selftest_ksint_forward(sb200_context *ctx, const uint64_t *h_rows, size_t rows, uint32_t *h_out)
{
    SB_NEED(ctx);
    SB_NEED(h_rows);
    SB_NEED(h_out);
    SB_TRY
    Context &c = *ctx->c;
    std::lock_guard<std::mutex> lock(c.mu);
    cuda_check(cudaSetDevice(c.device), "cudaSetDevice");
    ksint_selftest_transform(c, false, reinterpret_cast<const u64 *>(h_rows), rows, h_out);
    return SB200_OK;
    SB_CATCH
}

int sb200_selftest_ksint_inverse(sb200_context *ctx, uint32_t *h_data, size_t rows)
{
    SB_NEED(ctx);
    SB_NEED(h_data);
    SB_TRY
    Context &c = *ctx->c;
    std::lock_guard<std::mutex> lock(c.mu);
    cuda_check(cudaSetDevice(c.device), "cudaSetDevice");
    ksint_selftest_transform(c, true, nullptr, rows, h_data);
    return SB200_OK;
    SB_CATCH
}

int sb200_selftest_ksint_product(sb200_context *ctx, const uint32_t *h_Dh, const uint32_t *h_key, size_t L, size_t B, uint32_t *h_Acc,
                                 int kernel, int *ran)
{
    SB_NEED(ctx);
    SB_NEED(h_Dh);
    SB_NEED(h_key);
    SB_NEED(h_Acc);
    SB_TRY
    Context &c = *ctx->c;
    std::lock_guard<std::mutex> lock(c.mu);
    cuda_check(cudaSetDevice(c.device), "cudaSetDevice");
    if (L > 1024 || B > (size_t(1) << 20))
        throw std::invalid_argument("product: L or B out of range");
    const int r = ksint_selftest_product(c, h_Dh, h_key, static_cast<int>(L), static_cast<int>(B), h_Acc, kernel);
    if (ran)
        *ran = r;
    return SB200_OK;
    SB_CATCH
}

int sb200_selftest_rate(sb200_context *ctx, int kind, double *warp_ops_per_second)
{
    SB_NEED(warp_ops_per_second);
    SB_NEED(ctx);
    SB_TRY
    Context &c = *ctx->c;
    std::lock_guard<std::mutex> lock(c.mu);
    cuda_check(cudaSetDevice(c.device), "cudaSetDevice");
    *warp_ops_per_second = kind >= 10 ? ksint_selftest_rate(c, kind - 10, nullptr) : selftest_rate(c, kind, nullptr);
    return SB200_OK;
    SB_CATCH
}

int sb200_profile_read_work(sb200_context *ctx, size_t index, char *name, size_t name_capacity, double *total_ms,
                            unsigned long long *launches, double *algorithmic_bytes, double *butterflies, double *macs)
{
    return sb200_profile_read_work32(ctx, index, name, name_capacity, total_ms, launches, algorithmic_bytes, butterflies, macs, nullptr, nullptr);
}

int sb200_profile_read_work32(sb200_context *ctx, size_t index, char *name, size_t name_capacity, double *total_ms,
                              unsigned long long *launches, double *algorithmic_bytes, double *butterflies, double *macs,
                              double *butterflies32, double *macs32)
{
    SB_NEED(ctx);
    SB_NEED(name);
    SB_NEED(total_ms);
    SB_NEED(launches);
    SB_NEED(algorithmic_bytes);
    SB_TRY
    Context &c = *ctx->c;
    std::lock_guard<std::mutex> lock(c.mu);
    cuda_check(cudaSetDevice(c.device), "cudaSetDevice");
    cuda_check(cudaDeviceSynchronize(), "synchronize");
    // aggregate by (name, pass) in first-seen order
    struct Agg
    {
        std::string name;
        double ms = 0, bytes = 0, bflys = 0, macs = 0, bflys32 = 0, macs32 = 0;
        unsigned long long n = 0;
    };
    std::vector<Agg> aggs;
    static const char *suffix[] = { "", ":col", ":local" };
    for (auto &r : c.stats.recs)
    {
        std::string nm = std::string(r.name) + suffix[r.pass];
        float ms = 0;
        cuda_check(cudaEventElapsedTime(&ms, r.e0, r.e1), "cudaEventElapsedTime");
        auto it = std::find_if(aggs.begin(), aggs.end(), [&](const Agg &a) { return a.name == nm; });
        if (it == aggs.end())
        {
            aggs.push_back(Agg{ nm });
            it = aggs.end() - 1;
        }
        it->ms += ms, it->bytes += r.bytes, it->bflys += r.bflys, it->macs += r.macs, it->bflys32 += r.bflys32, it->macs32 += r.macs32, it->n++;
    }
    if (index >= aggs.size())
        throw std::out_of_range("profile index");
    std::snprintf(name, name_capacity, "%s", aggs[index].name.c_str());
    *total_ms = aggs[index].ms;
    *launches = aggs[index].n;
    *algorithmic_bytes = aggs[index].bytes;
    if (butterflies)
        *butterflies = aggs[index].bflys;
    if (macs)
        *macs = aggs[index].macs;
    if (butterflies32)
        *butterflies32 = aggs[index].bflys32;
    if (macs32)
        *macs32 = aggs[index].macs32;
    return SB200_OK;
    SB_CATCH
}

} // extern "C"

// A device key handle is built in two steps around filling its words: kswitch_key_alloc makes the handle with room for `digits`
// digits ([digits][2][k][n] at d_key); kswitch_key_finish then checks every word is below its modulus (is_data_valid_for,
// valcheck.cpp:412-456: the fused key-switch kernel relies on it to keep its 128-bit sums in range; false = out of range, the caller
// throws its own error) and prepares the integer key-switching path's copy of the key.
static std::unique_ptr<sb200_kswitch_key> kswitch_key_alloc(Context &c, size_t digits)
{
    auto h = std::make_unique<sb200_kswitch_key>();
    h->k.d_key = DevBuf<u64>(digits * 2 * c.k * c.n);
    h->k.ctx = &c;
    h->k.digits = digits;
    return h;
}

static bool kswitch_key_finish(Context &c, KSwitchKey &k)
{
    if (!op_residues_in_range(c, c.k, k.digits * 2 * c.k, k.d_key.get(), nullptr))
        return false;
    ksint_prepare_key(c, k, nullptr);
    return true;
}

extern "C" {
int sb200_kswitch_key_create(sb200_context *ctx, const uint64_t *h_key, size_t digits, sb200_kswitch_key **out)
{
    SB_NEED(ctx);
    SB_NEED(h_key);
    SB_NEED(out);
    SB_TRY
    Context &c = *ctx->c;
    if (c.k < 2)
        throw std::logic_error("keyswitching is not supported by the context");
    if (digits < 1 || digits > c.k - 1)
        throw std::invalid_argument("kswitch key has an invalid number of digits");
    std::lock_guard<std::mutex> lock(c.mu);
    cuda_check(cudaSetDevice(c.device), "cudaSetDevice");
    auto h = kswitch_key_alloc(c, digits);
    cuda_check(cudaMemcpy(h->k.d_key.get(), h_key, digits * 2 * c.k * c.n * sizeof(u64), cudaMemcpyHostToDevice), "upload key");
    if (!kswitch_key_finish(c, h->k))
        throw std::invalid_argument("kswitch key data is not valid for encryption parameters");
    *out = h.release();
    return SB200_OK;
    SB_CATCH
}

} // extern "C"

// KSwitchKeys::load of the entries data()[indices[i]] (indices == nullptr: every non-empty slot, at most `capacity` of them) in one
// pass: the object is inflated at most once and its frame parsed once, every argument and metadata check runs before the first
// handle is made, then each entry's rows go host -> device (c_0 only for a seeded member) and its seeded c_1s expand on the device.
// Returns the handles in the order of `slots`; if anything throws, the handles made so far are destroyed with the vector.
static std::vector<std::unique_ptr<sb200_kswitch_key>> kswitch_keys_load(Context &c, const uint8_t *stream, size_t len, const size_t *indices,
                                                                         size_t count, std::vector<size_t> &slots)
{
    if (c.k < 2)
        throw std::logic_error("keyswitching is not supported by the context");
    std::vector<sbw::KSwitchEntry> entries;
    std::vector<uint8_t> plain; // KSwitchKeys saved with compr_mode_type::zlib: inflate the object, then parse as usual
    // bound: a GaloisKeys object holds at most 2 log2(n) + 1 < 64 keys of k-1 digits, plus one size word per slot
    if (sbw::inflate_stream(stream, len, 64 * (c.k - 1) * sbw::save_size(2 * c.k * c.n) + 16 * c.n + 4096, plain))
        stream = plain.data(), len = plain.size();
    sbw::inspect_kswitch_slots(stream, len, indices, count, slots, entries);
    if (!indices && entries.size() > count)
        throw std::invalid_argument("out has too few entries for the keys present");
    for (const sbw::KSwitchEntry &e : entries)
    {
        // is_valid_for(KSwitchKeys): keys live at the key level of this context (valcheck.cpp, kswitchkeys.cpp:149-153)
        if (e.n != c.n || e.L != c.k || std::memcmp(e.parms_id, c.parms_ids[c.k - 1].data(), sizeof(e.parms_id)) != 0)
            throw std::logic_error("KSwitchKeys data is invalid");
        // is_valid_for(KSwitchKeys) (valcheck.cpp:292-323): one public key per decomposition prime, i.e. exactly k-1 digits
        if (e.offsets.size() != c.k - 1)
            throw std::logic_error("KSwitchKeys data is invalid");
    }
    const size_t digits = c.k - 1, row = 2 * c.k * c.n * sizeof(u64);
    std::lock_guard<std::mutex> lock(c.mu);
    cuda_check(cudaSetDevice(c.device), "cudaSetDevice");
    std::vector<std::unique_ptr<sb200_kswitch_key>> keys;
    keys.reserve(entries.size());
    for (const sbw::KSwitchEntry &e : entries)
    {
        keys.push_back(kswitch_key_alloc(c, digits));
        u64 *d_key = keys.back()->k.d_key.get();
        // a seed-compressed member carries c_0 only (k n words) and the seed of c_1 = sample_poly_uniform at the key level
        // (KSwitchKeys::load -> PublicKey::load -> Ciphertext::expand_seed, ciphertext.cpp:118-150)
        std::vector<u64> seeds;
        std::vector<int> types;
        std::vector<long long> seed_dst;
        for (size_t j = 0; j < digits; j++)
        {
            cuda_check(cudaMemcpy(reinterpret_cast<uint8_t *>(d_key) + j * row, stream + e.offsets[j], e.seeded[j] ? row / 2 : row,
                                  cudaMemcpyHostToDevice),
                       "upload key");
            if (e.seeded[j])
            {
                u64 sd[8];
                std::memcpy(sd, stream + e.seed_offsets[j], sizeof(sd));
                seeds.insert(seeds.end(), sd, sd + 8);
                types.push_back(e.seeded[j]);
                seed_dst.push_back(static_cast<long long>((2 * j + 1) * c.k * c.n));
            }
        }
        if (!seed_dst.empty())
            op_expand_seeded(c, c.k, seed_dst.size(), seeds.data(), types.data(), seed_dst.data(), d_key, nullptr);
        if (!kswitch_key_finish(c, keys.back()->k)) // KSwitchKeys::load ends in is_valid_for (kswitchkeys.cpp:149-153)
            throw std::logic_error("KSwitchKeys data is invalid");
    }
    return keys;
}

extern "C" {
int sb200_kswitch_key_load(sb200_context *ctx, const uint8_t *stream, size_t len, size_t index, sb200_kswitch_key **out)
{
    SB_NEED(ctx);
    SB_NEED(stream);
    SB_NEED(out);
    SB_TRY
    std::vector<size_t> slots;
    auto keys = kswitch_keys_load(*ctx->c, stream, len, &index, 1, slots);
    *out = keys[0].release();
    return SB200_OK;
    SB_CATCH
}

int sb200_kswitch_keys_load(sb200_context *ctx, const uint8_t *stream, size_t len, const size_t *indices, size_t count,
                            sb200_kswitch_key **out, size_t *out_indices, size_t *out_count)
{
    SB_NEED(ctx);
    SB_NEED(stream);
    SB_NEED(out);
    SB_NEED(out_count);
    SB_TRY
    std::vector<size_t> slots;
    auto keys = kswitch_keys_load(*ctx->c, stream, len, indices, count, slots);
    for (size_t i = 0; i < keys.size(); i++)
    {
        out[i] = keys[i].release();
        if (out_indices)
            out_indices[i] = slots[i];
    }
    *out_count = keys.size();
    return SB200_OK;
    SB_CATCH
}

size_t sb200_kswitch_key_device_bytes(const sb200_kswitch_key *key)
{
    return key ? key->k.d_key.bytes() + key->k.d_key32.bytes() : 0;
}

int sb200_kswitch_key_destroy(sb200_kswitch_key *key)
{
    SB_NEED(key);
    delete key;
    return SB200_OK;
}
} // extern "C"

#define SB_ENTER(ctx)                                      \
    SB_NEED(ctx);                                          \
    Context &c = *ctx->c;                                  \
    std::lock_guard<std::mutex> lock(c.mu);                \
    cuda_check(cudaSetDevice(c.device), "cudaSetDevice");

// The scratch arenas of a context are shared by all of its calls.  Calls on one stream are ordered by the stream; a call on a
// different stream than the previous one first waits for that one's work (one event record per call, no host synchronisation).
namespace
{
    struct StreamOrder
    {
        Context &c;
        cudaStream_t st;
        StreamOrder(Context &ctx, cudaStream_t stream) : c(ctx), st(stream)
        {
            if (!c.order_event)
                c.order_event = make_event();
            if (c.order_valid && c.order_stream != st)
                cuda_check(cudaStreamWaitEvent(st, c.order_event.get(), 0), "cudaStreamWaitEvent(order)");
        }
        ~StreamOrder()
        {
            if (cudaEventRecord(c.order_event.get(), st) == cudaSuccess)
                c.order_stream = st, c.order_valid = true;
        }
    };
} // namespace
#define SB_ENTER_STREAM(ctx, stream) \
    SB_ENTER(ctx)                    \
    StreamOrder order_(c, static_cast<cudaStream_t>(stream));

static void check_batch(size_t batch)
{
    if (batch == 0)
        throw std::invalid_argument("batch must be positive");
}

static void check_level(const Context &c, size_t L, size_t batch)
{
    if (L < 1 || L > c.k)
        throw std::invalid_argument("encrypted is not valid for encryption parameters");
    check_batch(batch);
}

static void check_size(size_t size)
{
    if (size < 1 || size > 16) // SEAL_CIPHERTEXT_SIZE_MAX (util/defines.h)
        throw std::invalid_argument("invalid ciphertext size");
}

// ---- evaluator operations, encoder and decryptor ---------------------------------------------------------------------
// Each operation is described once: what it checks, its Layout (the input and output slabs of one ciphertext), and the launch
// on a chunk of B ciphertexts starting at ciphertext b0, which takes the chunk's input and output slabs in the layout's order.
// Two drivers turn a description into its entry points: on_stream (device slabs, the whole batch in one launch on the caller's
// stream) and on_host (host buffers).  The host-buffer entry points cut the batch into chunks that flow through a 3-stage
// pipeline on three streams: H2D copy of chunk i+1 | kernels of chunk i | D2H copy of chunk i-1, double-buffered device staging
// owned by the context (PCIe is full duplex, so with pinned host buffers both copy directions overlap each other and the compute).
// Pageable host memory works too, the copies then serialise inside the driver.
namespace
{
    struct Slab // an input
    {
        size_t words;          // per ciphertext (0: none; the pointer may then be NULL)
        const char *noun;      // what the pointer and overlap errors call it
        bool in_place = false; // an output may sit exactly on it: the same start and the same bytes per ciphertext
        bool shared = false;   // one operand of `words` words for the whole batch (a plaintext shared by every ciphertext)
        bool optional = false; // may be NULL (the values of an empty CKKS vector); every other slab must be present
    };
    struct Out
    {
        size_t words;              // per ciphertext
        size_t unit = sizeof(u64); // bytes of one word (the noise budget returns one int per ciphertext)
    };
    struct Layout
    {
        std::vector<Slab> in;
        std::vector<Out> out;
        const char *name = nullptr;  // the operation the overlap errors name (nullptr: the one- and two-input operations)
        const char *alias = nullptr; // the error when an output is exactly an input it may not sit on (nullptr: the overlap error)
        bool in_place = false;       // the operation updates its one input (out = in): the host pipeline stages one buffer
    };
    using Ins = std::vector<const u64 *>; // the caller's slabs in the layout's order
    using Outs = std::vector<u64 *>;
    // The caller's slabs as an entry point names them: a short list, or one or two operand arrays (each array checked non-NULL by
    // the entry point).  Nothing is copied until the driver asks, inside its SB_TRY.
    struct InSlabs
    {
        std::initializer_list<const void *> few;
        const uint64_t *const *p = nullptr, *const *q = nullptr;
        size_t n = 0, m = 0;
        InSlabs(std::initializer_list<const void *> list) : few(list) {}
        InSlabs(const uint64_t *const *p_, size_t n_, const uint64_t *const *q_ = nullptr, size_t m_ = 0) : p(p_), q(q_), n(n_), m(m_) {}
        Ins get() const
        {
            Ins v;
            for (const void *x : few)
                v.push_back(static_cast<const u64 *>(x));
            for (size_t i = 0; i < n + m; i++)
                v.push_back(reinterpret_cast<const u64 *>(i < n ? p[i] : q[i - n]));
            return v;
        }
    };
    struct OutSlabs
    {
        std::initializer_list<void *> few;
        uint64_t *const *p = nullptr;
        size_t n = 0;
        OutSlabs(std::initializer_list<void *> list) : few(list) {}
        OutSlabs(uint64_t *const *p_, size_t n_) : p(p_), n(n_) {}
        Outs get() const
        {
            Outs v;
            for (void *x : few)
                v.push_back(static_cast<u64 *>(x));
            for (size_t i = 0; i < n; i++)
                v.push_back(reinterpret_cast<u64 *>(p[i]));
            return v;
        }
    };

    // one- and two-input operations: input a (and b) and one output, which may sit exactly on an input unless alias names the error
    Layout unary(size_t a, size_t out, const char *alias = nullptr)
    {
        return { { { a, "input a", !alias } }, { { out } }, nullptr, alias };
    }
    Layout binary(size_t a, size_t b, size_t out, const char *alias = nullptr)
    {
        Layout w = unary(a, out, alias);
        w.in.push_back({ b, "input b", !alias });
        return w;
    }

    struct HostPipe
    {
        Context &c;
        cudaStream_t s_in, s_comp, s_out;
        cudaEvent_t ev_in[2], ev_comp[2], ev_out[2];
        explicit HostPipe(Context &ctx) : c(ctx)
        {
            IoArena &io = c.io;
            for (auto *s : { &io.s_in, &io.s_comp, &io.s_out })
                if (!*s)
                    *s = make_stream();
            for (int i = 0; i < 2; i++)
                for (auto *e : { &io.ev_in[i], &io.ev_comp[i], &io.ev_out[i] })
                    if (!*e)
                        *e = make_event();
            s_in = io.s_in.get(), s_comp = io.s_comp.get(), s_out = io.s_out.get();
            for (int i = 0; i < 2; i++)
                ev_in[i] = io.ev_in[i].get(), ev_comp[i] = io.ev_comp[i].get(), ev_out[i] = io.ev_out[i].get();
        }
        template <class Op>
        void run(size_t batch, const Layout &w, const Ins &h_in, const Outs &h_out, const Op &op)
        {
            if (w.in_place && (w.in.size() != 1 || w.out.size() != 1 || w.in[0].words != w.out[0].words || w.out[0].unit != sizeof(u64)))
                throw std::logic_error("an in-place layout has one input and one output of the same words");
            StreamOrder order(c, s_comp); // the operation's kernels (and the scratch arenas they use) run on s_comp
            size_t per_ct = 0;            // staged bytes per ciphertext
            for (const Slab &s : w.in)
                per_ct += s.shared ? 0 : s.words * sizeof(u64);
            for (const Out &o : w.out)
                per_ct += w.in_place ? 0 : o.words * o.unit;
            size_t chunk = std::max<size_t>(1, std::min<size_t>(batch, c.host_stage_bytes / std::max<size_t>(per_ct, 1)));
            if (chunk >= batch && batch >= 4)
                chunk = (batch + 1) / 2; // at least two chunks so the copies overlap the kernels
            // A slot's staging: the per-ciphertext inputs of a chunk in buf[slot][0], its outputs in buf[slot][2] (in place: the
            // output is staged on its input); the shared inputs in buf[0][1], uploaded once ahead of the first chunk and never overwritten.  Each slab
            // starts at a 256-byte boundary.
            const auto place = [](size_t &end, size_t words) {
                const size_t at = (end + 31) & ~size_t(31);
                end = at + words;
                return at;
            };
            std::vector<size_t> in_at(w.in.size()), out_at(w.out.size());
            size_t in_words = 0, shared_words = 0, out_words = 0;
            for (size_t x = 0; x < w.in.size(); x++)
                in_at[x] = w.in[x].shared ? place(shared_words, w.in[x].words) : place(in_words, chunk * w.in[x].words);
            for (size_t y = 0; y < w.out.size(); y++)
                out_at[y] = place(out_words, (chunk * w.out[y].words * w.out[y].unit + sizeof(u64) - 1) / sizeof(u64));
            // size all staging before the pipeline starts: growth synchronises the device
            for (int slot = 0; slot < 2; slot++)
            {
                c.io.buf[slot][0].grow(in_words);
                if (!w.in_place)
                    c.io.buf[slot][2].grow(out_words);
            }
            if (shared_words)
                c.io.buf[0][1].grow(shared_words);
            std::vector<u64 *> din[2], dout[2];
            for (int slot = 0; slot < 2; slot++)
            {
                for (size_t x = 0; x < w.in.size(); x++)
                    din[slot].push_back(w.in[x].words ? (w.in[x].shared ? c.io.buf[0][1] : c.io.buf[slot][0]).get() + in_at[x] : nullptr);
                for (size_t y = 0; y < w.out.size(); y++)
                    dout[slot].push_back(w.in_place ? din[slot][0] : c.io.buf[slot][2].get() + out_at[y]);
            }
            for (size_t x = 0; x < w.in.size(); x++)
                if (w.in[x].shared && w.in[x].words)
                    cuda_check(cudaMemcpyAsync(din[0][x], h_in[x], w.in[x].words * sizeof(u64), cudaMemcpyHostToDevice, s_in), "H2D");
            size_t i = 0;
            for (size_t b0 = 0; b0 < batch; b0 += chunk, i++)
            {
                const size_t B = std::min(chunk, batch - b0);
                const int slot = static_cast<int>(i & 1);
                if (i >= 2)
                {
                    // inputs of this slot are free once its previous kernels finished (and, in place, once copied out)
                    cuda_check(cudaStreamWaitEvent(s_in, w.in_place ? ev_out[slot] : ev_comp[slot], 0), "wait");
                }
                for (size_t x = 0; x < w.in.size(); x++)
                {
                    const Slab &s = w.in[x];
                    if (s.words && !s.shared)
                        cuda_check(cudaMemcpyAsync(din[slot][x], h_in[x] + b0 * s.words, B * s.words * sizeof(u64),
                                                   cudaMemcpyHostToDevice, s_in),
                                   "H2D");
                }
                cuda_check(cudaEventRecord(ev_in[slot], s_in), "record");
                cuda_check(cudaStreamWaitEvent(s_comp, ev_in[slot], 0), "wait");
                if (i >= 2 && !w.in_place)
                    cuda_check(cudaStreamWaitEvent(s_comp, ev_out[slot], 0), "wait"); // output staging of this slot drained
                op(c, b0, B, din[slot].data(), dout[slot].data(), s_comp);
                cuda_check(cudaEventRecord(ev_comp[slot], s_comp), "record");
                cuda_check(cudaStreamWaitEvent(s_out, ev_comp[slot], 0), "wait");
                for (size_t y = 0; y < w.out.size(); y++)
                {
                    const size_t bytes = w.out[y].words * w.out[y].unit; // per ciphertext
                    cuda_check(cudaMemcpyAsync(reinterpret_cast<uint8_t *>(h_out[y]) + b0 * bytes, dout[slot][y], B * bytes, cudaMemcpyDeviceToHost, s_out),
                               "D2H");
                }
                cuda_check(cudaEventRecord(ev_out[slot], s_out), "record");
            }
            cuda_check(cudaStreamSynchronize(s_out), "synchronize");
            cuda_check(cudaStreamSynchronize(s_comp), "synchronize");
        }
    };

    struct Ntt
    {
        bool inverse;
        size_t L, size;
        void check(const Context &c, size_t batch) const { check_level(c, L, batch); }
        Layout layout(const Context &c) const
        {
            Layout w = unary(size * L * c.n, size * L * c.n);
            w.in_place = true;
            return w;
        }
        void operator()(Context &c, size_t, size_t B, const u64 *const *, u64 *const *outs, cudaStream_t st) const
        {
            op_ntt(c, inverse, L, size, B, outs[0], st);
        }
    };

    // two size-2 ciphertexts; square: b is a (one operand crosses the bus, the NTT-form schemes square with their own kernel when
    // op_ckks_multiply sees a == b)
    struct Multiply
    {
        size_t L;
        bool square;
        void check(const Context &c, size_t batch) const
        {
            check_level(c, L, batch);
            check_bfv_multiply_level(c, L);
        }
        Layout layout(const Context &c) const { return square ? unary(2 * L * c.n, 3 * L * c.n) : binary(2 * L * c.n, 2 * L * c.n, 3 * L * c.n); }
        void operator()(Context &c, size_t, size_t B, const u64 *const *ins, u64 *const *outs, cudaStream_t st) const
        {
            const u64 *b = square ? ins[0] : ins[1];
            if (c.scheme != SB200_SCHEME_BFV) // CKKS and BGV share the NTT-form tensor (evaluator.cpp:569-708, :710-841)
                op_ckks_multiply(c, L, B, ins[0], b, outs[0], st);
            else
                op_bfv_multiply(c, L, B, ins[0], b, outs[0], st);
        }
    };

    struct MultiplySized
    {
        size_t L, sa, sb;
        void check(const Context &c, size_t batch) const
        {
            check_level(c, L, batch);
            check_sizes(sa, sb);
            check_bfv_multiply_level(c, L);
        }
        Layout layout(const Context &c) const
        {
            return binary(sa * L * c.n, sb * L * c.n, (sa + sb - 1) * L * c.n, "multiply: the output slab must not alias an input slab");
        }
        void operator()(Context &c, size_t, size_t B, const u64 *const *ins, u64 *const *outs, cudaStream_t st) const
        {
            if (c.scheme != SB200_SCHEME_BFV)
                op_ckks_multiply(c, L, sa, sb, B, ins[0], ins[1], outs[0], st);
            else
                op_bfv_multiply(c, L, sa, sb, B, ins[0], ins[1], outs[0], st);
        }
    };

    struct Linear // mode 0: a + b, 1: a - b, 2: -a
    {
        int mode;
        size_t L, size;
        void check(const Context &c, size_t batch) const { check_level(c, L, batch); }
        Layout layout(const Context &c) const
        {
            const size_t w = size * L * c.n;
            return mode == 2 ? unary(w, w) : binary(w, w, w);
        }
        void operator()(Context &c, size_t, size_t B, const u64 *const *ins, u64 *const *outs, cudaStream_t st) const
        {
            op_linear(c, mode, L, size, B, ins[0], mode == 2 ? nullptr : ins[1], outs[0], st);
        }
    };

    // count operands of sizes[j] polynomials folded into one of the largest size (op_add_many).  The output may be operand 0 in
    // place when it has the output's size; it may not meet any other operand
    struct AddMany
    {
        size_t L, count;
        const size_t *sizes;
        const int *modes;
        const u64 *factors;
        size_t out_size() const
        {
            size_t s = 0;
            for (size_t j = 0; j < count; j++)
                s = std::max(s, sizes[j]);
            return s;
        }
        // the fold's own checks, and the factors a scaled step needs (SB200_E_POINTER) after every other check
        void check_fold(const Context &c, size_t batch) const
        {
            check_level(c, L, batch);
            if (count == 0)
                throw std::invalid_argument("encrypteds cannot be empty");
            for (size_t j = 0; j < count; j++)
                check_size(sizes[j]);
            for (size_t j = 1; j < count && modes; j++)
                if (modes[j - 1] < 0 || modes[j - 1] > 3)
                    throw std::invalid_argument("invalid add_many mode");
        }
        void need_factors() const
        {
            for (size_t j = 1; j < count && modes && !factors; j++)
                if (modes[j - 1] & SB200_FOLD_SCALED)
                    throw null_pointer("h_factors");
        }
        void check(const Context &c, size_t batch) const
        {
            check_fold(c, batch);
            need_factors();
        }
        Layout layout(const Context &c) const
        {
            Layout w{ {}, { { out_size() * L * c.n } }, "add_many", "add_many: the output slab must not alias an operand other than operand 0" };
            for (size_t j = 0; j < count; j++)
                w.in.push_back({ sizes[j] * L * c.n, "an operand", j == 0 });
            return w;
        }
        void operator()(Context &c, size_t, size_t B, const u64 *const *ins, u64 *const *outs, cudaStream_t st) const
        {
            std::vector<int> m(count ? count - 1 : 0, SB200_FOLD_ADD);
            if (modes)
                std::copy(modes, modes + m.size(), m.begin());
            op_add_many(c, L, B, count, sizes, ins, m.data(), factors, outs[0], st);
        }
    };

    // plain_count: one plaintext per ciphertext (batch) or one for the whole batch (1, a shared operand: Slab::shared).  The
    // older entry points, which take one plaintext per ciphertext, stay on the per-ciphertext path at every batch size (shared =
    // false, plain_count = batch); the _n entry points share the plaintext when plain_count = 1.
    void check_plain_count(size_t plain_count, size_t batch)
    {
        if (plain_count != 1 && plain_count != batch)
            throw std::invalid_argument("plain_count must be 1 or batch");
    }

    // inputs: K ciphertext operands, then M K plaintext operands; M outputs, each a fold over K terms of multiply_plain(ct_t,
    // plain_{j K + t}) (op_multiply_plain_sum).  The fold's modes and factors are AddMany's, and are checked by it.  No output may
    // meet an operand or another output.
    struct PlainSum
    {
        AddMany fold; // L, K, sizes, modes, factors
        size_t M;
        const size_t *plain_counts;
        bool ct_ntt, plain_ntt;
        size_t K() const { return fold.count; }
        // in the chain's order: multiply_plain's checks of every term (the plaintext counts), then add_many's (sizes, modes)
        void check(Context &c, size_t batch) const
        {
            check_level(c, fold.L, batch);
            if (K() == 0)
                throw std::invalid_argument("encrypteds cannot be empty");
            if (M == 0)
                throw std::invalid_argument("outputs cannot be empty");
            for (size_t j = 0; j < M * K(); j++)
                check_plain_count(plain_counts[j], batch);
            fold.check_fold(c, batch);
            if (!plain_ntt)
                plain_level(c, fold.L); // "unsupported operation for scheme type" for CKKS
            fold.need_factors();
        }
        Layout layout(const Context &c) const
        {
            const size_t poly = fold.L * c.n;
            Layout w{ {}, std::vector<Out>(M, Out{ fold.out_size() * poly }), "multiply_plain_sum" };
            for (size_t t = 0; t < K(); t++)
                w.in.push_back({ fold.sizes[t] * poly, "a ciphertext operand" });
            for (size_t x = 0; x < M * K(); x++)
                w.in.push_back({ plain_ntt ? poly : c.n, "a plaintext operand", false, plain_counts[x] == 1 });
            return w;
        }
        void operator()(Context &c, size_t, size_t B, const u64 *const *ins, u64 *const *outs, cudaStream_t st) const
        {
            std::vector<size_t> counts(M * K()); // of this chunk
            for (size_t x = 0; x < M * K(); x++)
                counts[x] = plain_counts[x] == 1 ? 1 : B;
            op_multiply_plain_sum(c, fold.L, B, K(), M, fold.sizes, ins, counts.data(), ins + K(), ct_ntt, plain_ntt, fold.modes, fold.factors,
                                  outs, st);
        }
    };

    // inputs: M K left-hand operands, then K right-hand ones, all of size 2; M outputs, each a fold over K terms of
    // multiply(lhs_{j K + t}, rhs_t) (op_multiply_sum).  The fold's modes and factors are AddMany's, checked by it on the products'
    // size 3.  No output may meet an operand or another output.
    struct MultiplySum
    {
        size_t L, K, M;
        const int *modes;
        const u64 *factors;
        // in the chain's order: multiply's checks of every term (the level, BFV's multiplication limit), then add_many's (modes)
        void check(const Context &c, size_t batch) const
        {
            check_level(c, L, batch);
            if (K == 0)
                throw std::invalid_argument("encrypteds cannot be empty");
            if (M == 0)
                throw std::invalid_argument("outputs cannot be empty");
            check_bfv_multiply_level(c, L);
            const std::vector<size_t> sizes(K, 3);
            AddMany{ L, K, sizes.data(), modes, factors }.check(c, batch);
        }
        Layout layout(const Context &c) const
        {
            Layout w{ std::vector<Slab>(M * K, Slab{ 2 * L * c.n, "a left-hand operand" }), std::vector<Out>(M, Out{ 3 * L * c.n }), "multiply_sum" };
            w.in.resize(M * K + K, Slab{ 2 * L * c.n, "a right-hand operand" });
            return w;
        }
        void operator()(Context &c, size_t, size_t B, const u64 *const *ins, u64 *const *outs, cudaStream_t st) const
        {
            op_multiply_sum(c, L, B, K, M, ins, ins + M * K, modes, factors, outs, st);
        }
    };

    // the plaintext operations: a ciphertext slab of ct words, which the output may overwrite in place, and plain_count plaintexts
    // of pw words
    Layout with_plain(size_t ct, size_t pw, bool shared)
    {
        return { { { ct, "input a", true }, { pw, "input b", !shared, shared } }, { { ct } }, nullptr,
                 shared ? "the shared plaintext must not alias the output slab" : nullptr };
    }

    struct MultiplyPlain // b: NTT-form plaintexts [plain_count][L][n]
    {
        size_t L, size, plain_count;
        bool shared;
        void check(const Context &c, size_t batch) const
        {
            check_level(c, L, batch);
            check_plain_count(plain_count, batch);
        }
        Layout layout(const Context &c) const { return with_plain(size * L * c.n, L * c.n, shared); }
        void operator()(Context &c, size_t, size_t B, const u64 *const *ins, u64 *const *outs, cudaStream_t st) const
        {
            op_multiply_plain(c, L, size, B, shared, ins[0], ins[1], outs[0], st);
        }
    };

    struct AddPlainNtt // CKKS: b: NTT-form plaintexts [plain_count][L][n], added to (subtracted from) c_0
    {
        size_t L, size, plain_count;
        bool shared;
        bool subtract;
        void check(const Context &c, size_t batch) const
        {
            check_level(c, L, batch);
            check_plain_count(plain_count, batch);
        }
        Layout layout(const Context &c) const { return with_plain(size * L * c.n, L * c.n, shared); }
        void operator()(Context &c, size_t, size_t B, const u64 *const *ins, u64 *const *outs, cudaStream_t st) const
        {
            op_add_plain_ntt(c, L, size, B, shared, subtract, ins[0], ins[1], outs[0], st);
        }
    };

    struct PlainToNtt // a: coefficient-form plaintexts [B][n]
    {
        size_t L;
        void check(const Context &c, size_t batch) const { check_level(c, L, batch); }
        Layout layout(const Context &c) const { return unary(c.n, L * c.n); }
        void operator()(Context &c, size_t, size_t B, const u64 *const *ins, u64 *const *outs, cudaStream_t st) const
        {
            op_plain_to_ntt(c, L, B, ins[0], nullptr, outs[0], st);
        }
    };

    struct MultiplyPlainCoeff // b: coefficient-form plaintexts [plain_count][n]
    {
        size_t L, size, plain_count;
        bool shared;
        bool ct_is_ntt;
        void check(const Context &c, size_t batch) const
        {
            check_level(c, L, batch);
            check_plain_count(plain_count, batch);
        }
        Layout layout(const Context &c) const { return with_plain(size * L * c.n, c.n, shared); }
        void operator()(Context &c, size_t, size_t B, const u64 *const *ins, u64 *const *outs, cudaStream_t st) const
        {
            op_multiply_plain_coeff(c, L, size, B, shared, ct_is_ntt, ins[0], ins[1], outs[0], st);
        }
    };

    // b: coefficient-form plaintexts [plain_count][n]; cf: BGV correction factors on the host, one per plaintext (NULL = 1)
    struct AddPlainCoeff
    {
        size_t L, size, plain_count;
        bool shared;
        bool subtract;
        const u64 *cf;
        void check(const Context &c, size_t batch) const
        {
            check_level(c, L, batch);
            check_plain_count(plain_count, batch);
        }
        Layout layout(const Context &c) const { return with_plain(size * L * c.n, c.n, shared); }
        void operator()(Context &c, size_t b0, size_t B, const u64 *const *ins, u64 *const *outs, cudaStream_t st) const
        {
            op_add_plain_coeff(c, L, size, B, shared, subtract, ins[0], ins[1], cf && !shared ? cf + b0 : cf, outs[0], st);
        }
    };

    struct BatchCodec // values [B][n] <-> coefficient-form plaintexts [B][n]
    {
        bool decode;
        void check(const Context &, size_t batch) const { check_batch(batch); }
        Layout layout(const Context &c) const { return unary(c.n, c.n); }
        void operator()(Context &c, size_t, size_t B, const u64 *const *ins, u64 *const *outs, cudaStream_t st) const
        {
            if (decode)
                op_batch_decode(c, B, ins[0], outs[0], st);
            else
                op_batch_encode(c, B, ins[0], outs[0], st);
        }
    };

    struct Relinearize
    {
        size_t L;
        const KSwitchKey &key;
        void check(const Context &c, size_t batch) const { check_level(c, L, batch); }
        Layout layout(const Context &c) const
        {
            return unary(3 * L * c.n, 2 * L * c.n, "relinearize: input and output slabs must not alias (different layouts)");
        }
        void operator()(Context &c, size_t, size_t B, const u64 *const *ins, u64 *const *outs, cudaStream_t st) const
        {
            op_relinearize(c, L, B, ins[0], key, outs[0], st);
        }
    };

    struct MultiplyRelinearize
    {
        size_t L;
        const KSwitchKey &key;
        void check(const Context &c, size_t batch) const
        {
            check_level(c, L, batch);
            check_bfv_multiply_level(c, L);
        }
        Layout layout(const Context &c) const { return binary(2 * L * c.n, 2 * L * c.n, 2 * L * c.n); }
        void operator()(Context &c, size_t, size_t B, const u64 *const *ins, u64 *const *outs, cudaStream_t st) const
        {
            op_multiply_relinearize(c, L, B, ins[0], ins[1], key, outs[0], st);
        }
    };

    struct RelinearizeSized // one step of relinearize_internal's loop: (c_0, c_1) += switch_key(c_{size-1}), size unchanged
    {
        size_t L, size;
        const KSwitchKey &key;
        void check(const Context &c, size_t batch) const
        {
            check_level(c, L, batch);
            check_size(size);
        }
        Layout layout(const Context &c) const
        {
            return unary(size * L * c.n, size * L * c.n, "relinearize: input and output slabs must not alias");
        }
        void operator()(Context &c, size_t, size_t B, const u64 *const *ins, u64 *const *outs, cudaStream_t st) const
        {
            op_relinearize_sized(c, L, size, B, ins[0], key, outs[0], st);
        }
    };

    struct ApplyGalois
    {
        size_t L;
        uint32_t elt;
        const KSwitchKey &key;
        void check(const Context &c, size_t batch) const { check_level(c, L, batch); }
        Layout layout(const Context &c) const { return unary(2 * L * c.n, 2 * L * c.n); }
        void operator()(Context &c, size_t, size_t B, const u64 *const *ins, u64 *const *outs, cudaStream_t st) const
        {
            op_apply_galois(c, L, B, ins[0], elt, key, outs[0], st);
        }
    };

    // out = b + apply_galois(a); out may be b, b may be a
    struct ApplyGaloisAdd
    {
        size_t L;
        uint32_t elt;
        const KSwitchKey &key;
        void check(const Context &c, size_t batch) const
        {
            check_level(c, L, batch);
            check_rotate_sum_args(c, L, 1, &elt, std::array<const KSwitchKey *, 1>{ &key }.data());
        }
        Layout layout(const Context &c) const
        {
            Layout w = binary(2 * L * c.n, 2 * L * c.n, 2 * L * c.n, "apply_galois_add: in and out must not alias");
            w.in[1].in_place = true;
            return w;
        }
        void operator()(Context &c, size_t, size_t B, const u64 *const *ins, u64 *const *outs, cudaStream_t st) const
        {
            op_apply_galois_add(c, L, B, ins[0], elt, key, ins[1], outs[0], st);
        }
    };

    // out = y_steps, y_{j+1} = y_j + apply_galois(y_j, elts[j]); out may be a.  A host chunk runs the whole chain once staged
    struct RotateSum
    {
        size_t L, steps;
        const uint32_t *elts;
        const KSwitchKey *const *keys;
        void check(const Context &c, size_t batch) const
        {
            check_level(c, L, batch);
            check_rotate_sum_args(c, L, steps, elts, keys);
        }
        Layout layout(const Context &c) const { return unary(2 * L * c.n, 2 * L * c.n); }
        void operator()(Context &c, size_t, size_t B, const u64 *const *ins, u64 *const *outs, cudaStream_t st) const
        {
            op_rotate_sum(c, L, B, ins[0], steps, elts, keys, outs[0], st);
        }
    };

    // the key handles of a rotate_sum call, after the pointer checks (SB200_E_POINTER on a NULL array or entry)
    int rotate_sum_keys(size_t steps, const uint32_t *elts, const sb200_kswitch_key *const *keys, std::vector<const KSwitchKey *> &out)
    {
        if (steps)
        {
            SB_NEED(elts);
            SB_NEED(keys);
        }
        for (size_t j = 0; j < steps; j++)
        {
            SB_NEED(keys[j]);
            out.push_back(&keys[j]->k);
        }
        return SB200_OK;
    }

    // out = c + b * apply_galois(a), b: NTT-form plaintexts [plain_count][L][n]; out may be c, c may be a.  The checks in the chain's
    // order: apply_galois's (level, element, key), then multiply_plain's (the plaintext count)
    struct ApplyGaloisMultiplyPlainAdd
    {
        size_t L, plain_count;
        uint32_t elt;
        const KSwitchKey &key;
        void check(const Context &c, size_t batch) const
        {
            check_level(c, L, batch);
            check_rotate_sum_args(c, L, 1, &elt, std::array<const KSwitchKey *, 1>{ &key }.data());
            check_plain_count(plain_count, batch);
        }
        Layout layout(const Context &c) const
        {
            const size_t poly = L * c.n;
            const bool shared = plain_count == 1;
            return { { { 2 * poly, "input a" }, { poly, "the plaintext", false, shared }, { 2 * poly, "the addend", true } },
                     { { 2 * poly } },
                     nullptr,
                     "apply_galois_multiply_plain_add: in and out must not alias" };
        }
        void operator()(Context &c, size_t, size_t B, const u64 *const *ins, u64 *const *outs, cudaStream_t st) const
        {
            op_apply_galois_multiply_plain_add(c, L, B, ins[0], elt, key, plain_count == 1, ins[1], ins[2], outs[0], st);
        }
    };

    // out = sum_t plains[t] * apply_galois(in, elts[t]) (op_diagonal_sum): input 0 is the ciphertext slab, inputs 1 .. count the
    // plaintexts (NTT form [L][n] or coefficient form [n] per plaintext, plain_counts[t] of them).  The output may not meet any input.
    struct DiagonalSum
    {
        size_t L, count;
        const uint32_t *elts;
        const KSwitchKey *const *keys;
        const size_t *plain_counts;
        bool plain_ntt;
        // in the chain's order: apply_galois's checks of every rotated term, multiply_plain's of every term (the plaintext counts and,
        // for coefficient-form plaintexts, the scheme), then add_many's (the term count)
        void check(Context &c, size_t batch) const
        {
            check_level(c, L, batch);
            check_diagonal_sum_args(c, L, count, elts, keys);
            for (size_t t = 0; t < count; t++)
                check_plain_count(plain_counts[t], batch);
            if (!plain_ntt && count)
                plain_level(c, L); // "unsupported operation for scheme type" for CKKS
            if (count == 0)
                throw std::invalid_argument("encrypteds cannot be empty");
        }
        Layout layout(const Context &c) const
        {
            const size_t poly = L * c.n;
            Layout w{ { { 2 * poly, "input" } }, { { 2 * poly } }, "diagonal_sum", "diagonal_sum: in and out must not alias" };
            for (size_t t = 0; t < count; t++)
                w.in.push_back({ plain_ntt ? poly : c.n, "a plaintext operand", false, plain_counts[t] == 1 });
            return w;
        }
        void operator()(Context &c, size_t, size_t B, const u64 *const *ins, u64 *const *outs, cudaStream_t st) const
        {
            std::vector<size_t> counts(count); // of this chunk
            for (size_t t = 0; t < count; t++)
                counts[t] = plain_counts[t] == 1 ? 1 : B;
            op_diagonal_sum(c, L, B, ins[0], count, elts, keys, counts.data(), ins + 1, plain_ntt, outs[0], st);
        }
    };

    // the key handles of a diagonal_sum call, after the pointer checks (SB200_E_POINTER on a NULL array, or a NULL key of a rotated
    // term; element 1 needs none)
    int diagonal_sum_keys(size_t count, const uint32_t *elts, const sb200_kswitch_key *const *keys, const size_t *plain_counts,
                          const uint64_t *const *plains, std::vector<const KSwitchKey *> &out)
    {
        SB_NEED(elts);
        SB_NEED(keys);
        SB_NEED(plain_counts);
        SB_NEED(plains);
        for (size_t t = 0; t < count; t++)
        {
            if (elts[t] != 1)
                SB_NEED(keys[t]);
            out.push_back(keys[t] ? &keys[t]->k : nullptr);
        }
        return SB200_OK;
    }

    struct ModSwitch // rescale_to_next (CKKS) or mod_switch_to_next of ciphertexts of any size: L primes -> L - 1
    {
        bool rescale;
        size_t L, size;
        void check(const Context &c, size_t batch) const
        {
            check_level(c, L, batch);
            check_size(size);
            if (L < 2) // before the scheme, as the reference checks it (evaluator.cpp:1521, :1533)
                throw std::invalid_argument("end of modulus switching chain reached");
        }
        Layout layout(const Context &c) const
        {
            return unary(size * L * c.n, size * (L - 1) * c.n,
                         rescale ? "rescale_to_next: input and output slabs must not alias (different layouts)"
                                 : "mod_switch_to_next: input and output slabs must not alias (different layouts)");
        }
        void operator()(Context &c, size_t, size_t B, const u64 *const *ins, u64 *const *outs, cudaStream_t st) const
        {
            if (rescale)
                op_rescale(c, L, B * size, ins[0], outs[0], st);
            else
                op_mod_switch(c, L, B * size, ins[0], outs[0], st);
        }
    };

    // a: values, count doubles (reals) or count (re, im) pairs per plaintext; may be NULL, an error of check unless count = 0
    struct CkksEncode
    {
        size_t L, count;
        bool is_complex, has_values;
        double scale;
        void check(const Context &c, size_t batch) const
        {
            check_level(c, L, batch);
            if (count && !has_values)
                throw std::invalid_argument("values cannot be null");
        }
        Layout layout(const Context &c) const
        {
            Layout w = unary(count * (is_complex ? 2 : 1), L * c.n);
            w.in[0].optional = true;
            return w;
        }
        void operator()(Context &c, size_t, size_t B, const u64 *const *ins, u64 *const *outs, cudaStream_t st) const
        {
            op_ckks_encode(c, L, B, reinterpret_cast<const double *>(ins[0]), count, is_complex, scale, outs[0], st);
        }
    };

    // a: one scalar per plaintext, one word (real, int64) or two (complex).  h_values: the host entry point's values, checked in full
    // before the first chunk is staged, so that an error leaves h_plain untouched; the stream entry point checks inside the op
    struct CkksEncodeScalar
    {
        size_t L;
        int kind;
        double scale;
        const u64 *h_values;
        void check(const Context &c, size_t batch) const
        {
            check_ckks_scalar(c, L, kind, scale);
            check_batch(batch);
            if (h_values)
                check_ckks_scalar_values(c, L, batch, kind, h_values, scale);
        }
        Layout layout(const Context &c) const { return unary(kind == kCkksScalarComplex ? 2 : 1, L * c.n); }
        void operator()(Context &c, size_t, size_t B, const u64 *const *ins, u64 *const *outs, cudaStream_t st) const
        {
            op_ckks_encode_scalar(c, L, B, kind, ins[0], scale, outs[0], st);
        }
    };

    struct CkksDecode // out: n / 2 complex values (n doubles) per plaintext
    {
        size_t L;
        double scale;
        void check(const Context &c, size_t batch) const { check_level(c, L, batch); }
        Layout layout(const Context &c) const { return unary(L * c.n, c.n); }
        void operator()(Context &c, size_t, size_t B, const u64 *const *ins, u64 *const *outs, cudaStream_t st) const
        {
            op_ckks_decode(c, L, B, ins[0], scale, reinterpret_cast<double *>(outs[0]), st);
        }
    };

    struct Decrypt // out: CKKS NTT-form plaintexts [B][L][n], BFV / BGV coefficient-form plaintexts [B][n]; cf as in AddPlainCoeff
    {
        SecretKey &key;
        size_t L, size;
        const u64 *cf;
        void check(const Context &c, size_t batch) const { check_level(c, L, batch); }
        Layout layout(const Context &c) const { return unary(size * L * c.n, c.scheme == SB200_SCHEME_CKKS ? L * c.n : c.n); }
        void operator()(Context &c, size_t b0, size_t B, const u64 *const *ins, u64 *const *outs, cudaStream_t st) const
        {
            op_decrypt(c, key, L, size, B, ins[0], cf ? cf + b0 : nullptr, outs[0], st);
        }
    };

    // budgets: one int per ciphertext (Out::unit); ciphertexts in the scheme's own form (BFV coefficient, BGV NTT)
    struct NoiseBudget
    {
        SecretKey &key;
        size_t L, size;
        void check(const Context &c, size_t batch) const
        {
            check_level(c, L, batch);
            check_noise_budget(c, key, L, size);
        }
        Layout layout(const Context &c) const
        {
            Layout w = unary(size * L * c.n, 1);
            w.out[0].unit = sizeof(int);
            return w;
        }
        void operator()(Context &c, size_t, size_t B, const u64 *const *ins, u64 *const *outs, cudaStream_t st) const
        {
            op_invariant_noise_budget(c, key, L, size, B, ins[0], reinterpret_cast<int *>(outs[0]), st);
        }
    };

    // an entry point's own last step, inside its lock and stream order (the decryption wipes)
    using Then = void (*)(Context &c, cudaStream_t st);

    // what the errors call input x: its noun and, in a several-operand layout, its index in the caller's array of that noun
    std::string slab_name(const Layout &w, size_t x)
    {
        std::string s = w.in[x].noun;
        if (w.name)
        {
            size_t i = 0;
            for (size_t u = 0; u < x; u++)
                i += std::strcmp(w.in[u].noun, w.in[x].noun) == 0;
            s += " [" + std::to_string(i) + "]";
        }
        return s;
    }

    // every slab is present but an optional input
    void need_slabs(const Layout &w, const Ins &ins, const Outs &outs)
    {
        if (ins.size() != w.in.size() || outs.size() != w.out.size())
            throw std::logic_error("the slabs do not match the operation's layout");
        for (size_t x = 0; x < ins.size(); x++)
            if (!ins[x] && !w.in[x].optional)
                throw null_pointer(slab_name(w, x));
        for (size_t y = 0; y < outs.size(); y++)
            if (!outs[y])
                throw null_pointer(w.name ? "output slab [" + std::to_string(y) + "]" : "output slab");
    }

    // Device slabs: an output's byte range may meet an input's only where the input allows the output in place, and then only
    // where every ciphertext's output sits where its input was: same start and same bytes per ciphertext.  It may not meet another
    // output's.  Any other overlap lets one thread overwrite words another thread has still to read.  An output on an in-place
    // input with different words per ciphertext is refused for one ciphertext too: some kernels would be safe there (the 2 x 2
    // tensor reads a coefficient's words before writing them), others not (PlainToNtt, n -> L n words: row i > 0 reads the
    // plaintext words that row 0 overwrites), and the rule does not depend on which.
    void check_overlap(const Layout &w, size_t batch, const Ins &ins, const Outs &outs)
    {
        auto meet = [](const void *x, size_t nx, const void *y, size_t ny) {
            const auto *p = static_cast<const uint8_t *>(x), *q = static_cast<const uint8_t *>(y);
            return nx && ny && p < q + ny && q < p + nx;
        };
        if (w.alias) // an output exactly on an input it may not sit on: the operation's own error, ahead of any other overlap
            for (const void *o : outs)
                for (size_t x = 0; x < ins.size(); x++)
                    if (o == ins[x] && !w.in[x].in_place)
                        throw std::invalid_argument(w.alias);
        const auto op = [&] { return w.name ? std::string(w.name) + ": " : std::string(); }; // the messages are built when thrown
        for (size_t y = 0; y < outs.size(); y++)
        {
            const size_t stride = w.out[y].words * w.out[y].unit;
            for (size_t x = 0; x < ins.size(); x++)
            {
                const Slab &s = w.in[x];
                const size_t in_stride = s.shared ? 0 : s.words * sizeof(u64);
                if (!meet(outs[y], batch * stride, ins[x], s.shared ? s.words * sizeof(u64) : batch * in_stride))
                    continue;
                if (outs[y] == ins[x] && s.in_place && stride == in_stride)
                    continue;
                throw std::invalid_argument(op() + (w.out.size() > 1 ? "an" : "the") + " output slab must not overlap " + slab_name(w, x) +
                                            (s.in_place ? " other than exactly in place" : ""));
            }
            for (size_t u = 0; u < y; u++)
                if (meet(outs[y], batch * stride, outs[u], batch * w.out[u].words * w.out[u].unit))
                    throw std::invalid_argument(op() + "output slabs must not overlap");
        }
    }

    // The checks of both drivers, in this order: the slab pointers, then (with the context entered) the operation's own, then the
    // overlap rule: on device slabs always; on host buffers for the several-operand operations, whose outputs the pipeline could
    // otherwise copy back over host words a later chunk has still to upload.  The one- and two-input operations keep accepting
    // overlapping host buffers, as they always have.
    template <class Op>
    int on_stream(sb200_context *ctx, void *stream, size_t batch, const InSlabs &in, const OutSlabs &out, const Op &op, Then then = nullptr)
    {
        SB_NEED(ctx);
        SB_TRY
        const Layout w = op.layout(*ctx->c);
        const Ins ins = in.get();
        const Outs outs = out.get();
        need_slabs(w, ins, outs);
        SB_ENTER_STREAM(ctx, stream)
        op.check(c, batch);
        check_overlap(w, batch, ins, outs);
        auto st = static_cast<cudaStream_t>(stream);
        op(c, 0, batch, ins.data(), outs.data(), st);
        if (then)
            then(c, st);
        return SB200_OK;
        SB_CATCH
    }

    template <class Op>
    int on_host(sb200_context *ctx, size_t batch, const InSlabs &in, const OutSlabs &out, const Op &op, Then then = nullptr)
    {
        SB_NEED(ctx);
        SB_TRY
        const Layout w = op.layout(*ctx->c);
        const Ins ins = in.get();
        const Outs outs = out.get();
        need_slabs(w, ins, outs);
        SB_ENTER(ctx)
        op.check(c, batch);
        if (w.name)
            check_overlap(w, batch, ins, outs);
        HostPipe(c).run(batch, w, ins, outs, op);
        if (then)
            then(c, c.io.s_comp.get());
        return SB200_OK;
        SB_CATCH
    }

} // namespace

extern "C" {

int sb200_ntt_forward(sb200_context *ctx, size_t L, size_t size, size_t batch, uint64_t *d, void *stream)
{
    return on_stream(ctx, stream, batch, { d }, { d }, Ntt{ false, L, size });
}
int sb200_ntt_forward_host(sb200_context *ctx, size_t L, size_t size, size_t batch, uint64_t *h)
{
    return on_host(ctx, batch, { h }, { h }, Ntt{ false, L, size });
}
int sb200_ntt_inverse(sb200_context *ctx, size_t L, size_t size, size_t batch, uint64_t *d, void *stream)
{
    return on_stream(ctx, stream, batch, { d }, { d }, Ntt{ true, L, size });
}
int sb200_ntt_inverse_host(sb200_context *ctx, size_t L, size_t size, size_t batch, uint64_t *h)
{
    return on_host(ctx, batch, { h }, { h }, Ntt{ true, L, size });
}

int sb200_multiply(sb200_context *ctx, size_t L, size_t batch, const uint64_t *a, const uint64_t *b, uint64_t *out3, void *stream)
{
    return on_stream(ctx, stream, batch, { a, b }, { out3 }, Multiply{ L, false });
}
int sb200_multiply_host(sb200_context *ctx, size_t L, size_t batch, const uint64_t *a, const uint64_t *b, uint64_t *out3)
{
    return on_host(ctx, batch, { a, b }, { out3 }, Multiply{ L, false });
}
int sb200_square(sb200_context *ctx, size_t L, size_t batch, const uint64_t *a, uint64_t *out3, void *stream)
{
    return on_stream(ctx, stream, batch, { a }, { out3 }, Multiply{ L, true });
}
int sb200_square_host(sb200_context *ctx, size_t L, size_t batch, const uint64_t *a, uint64_t *out3)
{
    return on_host(ctx, batch, { a }, { out3 }, Multiply{ L, true });
}

int sb200_multiply_sized(sb200_context *ctx, size_t L, size_t size_a, size_t size_b, size_t batch, const uint64_t *a, const uint64_t *b,
                         uint64_t *out, void *stream)
{
    return on_stream(ctx, stream, batch, { a, b }, { out }, MultiplySized{ L, size_a, size_b });
}
int sb200_multiply_sized_host(sb200_context *ctx, size_t L, size_t size_a, size_t size_b, size_t batch, const uint64_t *a, const uint64_t *b,
                              uint64_t *out)
{
    return on_host(ctx, batch, { a, b }, { out }, MultiplySized{ L, size_a, size_b });
}

int sb200_add(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *a, const uint64_t *b, uint64_t *out, void *stream)
{
    return on_stream(ctx, stream, batch, { a, b }, { out }, Linear{ 0, L, size });
}
int sb200_add_host(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *a, const uint64_t *b, uint64_t *out)
{
    return on_host(ctx, batch, { a, b }, { out }, Linear{ 0, L, size });
}
int sb200_sub(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *a, const uint64_t *b, uint64_t *out, void *stream)
{
    return on_stream(ctx, stream, batch, { a, b }, { out }, Linear{ 1, L, size });
}
int sb200_sub_host(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *a, const uint64_t *b, uint64_t *out)
{
    return on_host(ctx, batch, { a, b }, { out }, Linear{ 1, L, size });
}
int sb200_negate(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *a, uint64_t *out, void *stream)
{
    return on_stream(ctx, stream, batch, { a }, { out }, Linear{ 2, L, size });
}
int sb200_negate_host(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *a, uint64_t *out)
{
    return on_host(ctx, batch, { a }, { out }, Linear{ 2, L, size });
}

int sb200_add_many(sb200_context *ctx, size_t L, size_t batch, size_t count, const size_t *sizes, const uint64_t *const *ops, const int *modes,
                   const uint64_t *factors, uint64_t *out, void *stream)
{
    SB_NEED(sizes);
    SB_NEED(ops);
    return on_stream(ctx, stream, batch, InSlabs(ops, count), { out }, AddMany{ L, count, sizes, modes, reinterpret_cast<const u64 *>(factors) });
}
int sb200_add_many_host(sb200_context *ctx, size_t L, size_t batch, size_t count, const size_t *sizes, const uint64_t *const *ops, const int *modes,
                        const uint64_t *factors, uint64_t *out)
{
    SB_NEED(sizes);
    SB_NEED(ops);
    return on_host(ctx, batch, InSlabs(ops, count), { out }, AddMany{ L, count, sizes, modes, reinterpret_cast<const u64 *>(factors) });
}

int sb200_multiply_plain_sum(sb200_context *ctx, size_t L, size_t batch, size_t count, size_t outputs, const size_t *sizes,
                             const uint64_t *const *cts, const size_t *plain_counts, const uint64_t *const *plains, int ct_is_ntt,
                             int plain_is_ntt, const int *modes, const uint64_t *factors, uint64_t *const *outs, void *stream)
{
    SB_NEED(sizes);
    SB_NEED(plain_counts);
    SB_NEED(cts);
    SB_NEED(plains);
    SB_NEED(outs);
    return on_stream(ctx, stream, batch, InSlabs(cts, count, plains, outputs * count), OutSlabs(outs, outputs),
                     PlainSum{ AddMany{ L, count, sizes, modes, reinterpret_cast<const u64 *>(factors) }, outputs, plain_counts, ct_is_ntt != 0,
                               plain_is_ntt != 0 });
}
int sb200_multiply_plain_sum_host(sb200_context *ctx, size_t L, size_t batch, size_t count, size_t outputs, const size_t *sizes,
                                  const uint64_t *const *cts, const size_t *plain_counts, const uint64_t *const *plains, int ct_is_ntt,
                                  int plain_is_ntt, const int *modes, const uint64_t *factors, uint64_t *const *outs)
{
    SB_NEED(sizes);
    SB_NEED(plain_counts);
    SB_NEED(cts);
    SB_NEED(plains);
    SB_NEED(outs);
    return on_host(ctx, batch, InSlabs(cts, count, plains, outputs * count), OutSlabs(outs, outputs),
                   PlainSum{ AddMany{ L, count, sizes, modes, reinterpret_cast<const u64 *>(factors) }, outputs, plain_counts, ct_is_ntt != 0,
                             plain_is_ntt != 0 });
}

int sb200_multiply_sum(sb200_context *ctx, size_t L, size_t batch, size_t count, size_t outputs, const uint64_t *const *lhs,
                       const uint64_t *const *rhs, const int *modes, const uint64_t *factors, uint64_t *const *outs, void *stream)
{
    SB_NEED(lhs);
    SB_NEED(rhs);
    SB_NEED(outs);
    return on_stream(ctx, stream, batch, InSlabs(lhs, outputs * count, rhs, count), OutSlabs(outs, outputs),
                     MultiplySum{ L, count, outputs, modes, reinterpret_cast<const u64 *>(factors) });
}
int sb200_multiply_sum_host(sb200_context *ctx, size_t L, size_t batch, size_t count, size_t outputs, const uint64_t *const *lhs,
                            const uint64_t *const *rhs, const int *modes, const uint64_t *factors, uint64_t *const *outs)
{
    SB_NEED(lhs);
    SB_NEED(rhs);
    SB_NEED(outs);
    return on_host(ctx, batch, InSlabs(lhs, outputs * count, rhs, count), OutSlabs(outs, outputs),
                   MultiplySum{ L, count, outputs, modes, reinterpret_cast<const u64 *>(factors) });
}

int sb200_multiply_plain(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *a, const uint64_t *plain, uint64_t *out,
                         void *stream)
{
    return on_stream(ctx, stream, batch, { a, plain }, { out }, MultiplyPlain{ L, size, batch, false });
}
int sb200_multiply_plain_host(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *a, const uint64_t *plain, uint64_t *out)
{
    return on_host(ctx, batch, { a, plain }, { out }, MultiplyPlain{ L, size, batch, false });
}
int sb200_multiply_plain_n(sb200_context *ctx, size_t L, size_t size, size_t batch, size_t plain_count, const uint64_t *a, const uint64_t *plain,
                           uint64_t *out, void *stream)
{
    return on_stream(ctx, stream, batch, { a, plain }, { out }, MultiplyPlain{ L, size, plain_count, plain_count == 1 });
}
int sb200_multiply_plain_n_host(sb200_context *ctx, size_t L, size_t size, size_t batch, size_t plain_count, const uint64_t *a,
                                const uint64_t *plain, uint64_t *out)
{
    return on_host(ctx, batch, { a, plain }, { out }, MultiplyPlain{ L, size, plain_count, plain_count == 1 });
}

int sb200_add_plain_ntt(sb200_context *ctx, size_t L, size_t size, size_t batch, size_t plain_count, int subtract, const uint64_t *a,
                        const uint64_t *plain, uint64_t *out, void *stream)
{
    return on_stream(ctx, stream, batch, { a, plain }, { out }, AddPlainNtt{ L, size, plain_count, plain_count == 1, subtract != 0 });
}
int sb200_add_plain_ntt_host(sb200_context *ctx, size_t L, size_t size, size_t batch, size_t plain_count, int subtract, const uint64_t *a,
                             const uint64_t *plain, uint64_t *out)
{
    return on_host(ctx, batch, { a, plain }, { out }, AddPlainNtt{ L, size, plain_count, plain_count == 1, subtract != 0 });
}

int sb200_plain_to_ntt(sb200_context *ctx, size_t L, size_t batch, const uint64_t *plain, uint64_t *out, void *stream)
{
    return on_stream(ctx, stream, batch, { plain }, { out }, PlainToNtt{ L });
}
int sb200_plain_to_ntt_host(sb200_context *ctx, size_t L, size_t batch, const uint64_t *plain, uint64_t *out)
{
    return on_host(ctx, batch, { plain }, { out }, PlainToNtt{ L });
}

int sb200_multiply_plain_coeff(sb200_context *ctx, size_t L, size_t size, size_t batch, int ct_is_ntt, const uint64_t *a, const uint64_t *plain,
                               uint64_t *out, void *stream)
{
    return on_stream(ctx, stream, batch, { a, plain }, { out }, MultiplyPlainCoeff{ L, size, batch, false, ct_is_ntt != 0 });
}
int sb200_multiply_plain_coeff_host(sb200_context *ctx, size_t L, size_t size, size_t batch, int ct_is_ntt, const uint64_t *a,
                                    const uint64_t *plain, uint64_t *out)
{
    return on_host(ctx, batch, { a, plain }, { out }, MultiplyPlainCoeff{ L, size, batch, false, ct_is_ntt != 0 });
}
int sb200_multiply_plain_coeff_n(sb200_context *ctx, size_t L, size_t size, size_t batch, size_t plain_count, int ct_is_ntt, const uint64_t *a,
                                 const uint64_t *plain, uint64_t *out, void *stream)
{
    return on_stream(ctx, stream, batch, { a, plain }, { out }, MultiplyPlainCoeff{ L, size, plain_count, plain_count == 1, ct_is_ntt != 0 });
}
int sb200_multiply_plain_coeff_n_host(sb200_context *ctx, size_t L, size_t size, size_t batch, size_t plain_count, int ct_is_ntt,
                                      const uint64_t *a, const uint64_t *plain, uint64_t *out)
{
    return on_host(ctx, batch, { a, plain }, { out }, MultiplyPlainCoeff{ L, size, plain_count, plain_count == 1, ct_is_ntt != 0 });
}

int sb200_add_plain_coeff(sb200_context *ctx, size_t L, size_t size, size_t batch, int subtract, const uint64_t *a, const uint64_t *plain,
                          const uint64_t *h_correction_factors, uint64_t *out, void *stream)
{
    return on_stream(ctx, stream, batch, { a, plain }, { out }, AddPlainCoeff{ L, size, batch, false, subtract != 0, (const u64 *)h_correction_factors });
}
int sb200_add_plain_coeff_host(sb200_context *ctx, size_t L, size_t size, size_t batch, int subtract, const uint64_t *a, const uint64_t *plain,
                               const uint64_t *h_correction_factors, uint64_t *out)
{
    return on_host(ctx, batch, { a, plain }, { out }, AddPlainCoeff{ L, size, batch, false, subtract != 0, (const u64 *)h_correction_factors });
}
int sb200_add_plain_coeff_n(sb200_context *ctx, size_t L, size_t size, size_t batch, size_t plain_count, int subtract, const uint64_t *a,
                            const uint64_t *plain, const uint64_t *h_correction_factors, uint64_t *out, void *stream)
{
    return on_stream(ctx, stream, batch, { a, plain }, { out }, AddPlainCoeff{ L, size, plain_count, plain_count == 1, subtract != 0, (const u64 *)h_correction_factors });
}
int sb200_add_plain_coeff_n_host(sb200_context *ctx, size_t L, size_t size, size_t batch, size_t plain_count, int subtract, const uint64_t *a,
                                 const uint64_t *plain, const uint64_t *h_correction_factors, uint64_t *out)
{
    return on_host(ctx, batch, { a, plain }, { out }, AddPlainCoeff{ L, size, plain_count, plain_count == 1, subtract != 0, (const u64 *)h_correction_factors });
}

int sb200_batch_encode(sb200_context *ctx, size_t batch, const uint64_t *values, uint64_t *plain, void *stream)
{
    return on_stream(ctx, stream, batch, { values }, { plain }, BatchCodec{ false });
}
int sb200_batch_encode_host(sb200_context *ctx, size_t batch, const uint64_t *values, uint64_t *plain)
{
    return on_host(ctx, batch, { values }, { plain }, BatchCodec{ false });
}
int sb200_batch_decode(sb200_context *ctx, size_t batch, const uint64_t *plain, uint64_t *values, void *stream)
{
    return on_stream(ctx, stream, batch, { plain }, { values }, BatchCodec{ true });
}
int sb200_batch_decode_host(sb200_context *ctx, size_t batch, const uint64_t *plain, uint64_t *values)
{
    return on_host(ctx, batch, { plain }, { values }, BatchCodec{ true });
}

int sb200_relinearize(sb200_context *ctx, size_t L, size_t batch, const uint64_t *in3, const sb200_kswitch_key *key, uint64_t *out2,
                      void *stream)
{
    SB_NEED(key);
    return on_stream(ctx, stream, batch, { in3 }, { out2 }, Relinearize{ L, key->k });
}
int sb200_relinearize_host(sb200_context *ctx, size_t L, size_t batch, const uint64_t *in3, const sb200_kswitch_key *key, uint64_t *out2)
{
    SB_NEED(key);
    return on_host(ctx, batch, { in3 }, { out2 }, Relinearize{ L, key->k });
}

int sb200_multiply_relinearize(sb200_context *ctx, size_t L, size_t batch, const uint64_t *a, const uint64_t *b,
                               const sb200_kswitch_key *key, uint64_t *out2, void *stream)
{
    SB_NEED(key);
    return on_stream(ctx, stream, batch, { a, b }, { out2 }, MultiplyRelinearize{ L, key->k });
}
int sb200_multiply_relinearize_host(sb200_context *ctx, size_t L, size_t batch, const uint64_t *a, const uint64_t *b,
                                    const sb200_kswitch_key *key, uint64_t *out2)
{
    SB_NEED(key);
    return on_host(ctx, batch, { a, b }, { out2 }, MultiplyRelinearize{ L, key->k });
}

int sb200_rescale_to_next_sized(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *in, uint64_t *out, void *stream)
{
    return on_stream(ctx, stream, batch, { in }, { out }, ModSwitch{ true, L, size });
}
int sb200_rescale_to_next_sized_host(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *in, uint64_t *out)
{
    return on_host(ctx, batch, { in }, { out }, ModSwitch{ true, L, size });
}
int sb200_rescale_to_next(sb200_context *ctx, size_t L, size_t batch, const uint64_t *in2, uint64_t *out2, void *stream)
{
    return on_stream(ctx, stream, batch, { in2 }, { out2 }, ModSwitch{ true, L, 2 });
}
int sb200_rescale_to_next_host(sb200_context *ctx, size_t L, size_t batch, const uint64_t *in2, uint64_t *out2)
{
    return on_host(ctx, batch, { in2 }, { out2 }, ModSwitch{ true, L, 2 });
}
int sb200_mod_switch_to_next_sized(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *in, uint64_t *out, void *stream)
{
    return on_stream(ctx, stream, batch, { in }, { out }, ModSwitch{ false, L, size });
}
int sb200_mod_switch_to_next_sized_host(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *in, uint64_t *out)
{
    return on_host(ctx, batch, { in }, { out }, ModSwitch{ false, L, size });
}
int sb200_mod_switch_to_next(sb200_context *ctx, size_t L, size_t batch, const uint64_t *in2, uint64_t *out2, void *stream)
{
    return on_stream(ctx, stream, batch, { in2 }, { out2 }, ModSwitch{ false, L, 2 });
}
int sb200_mod_switch_to_next_host(sb200_context *ctx, size_t L, size_t batch, const uint64_t *in2, uint64_t *out2)
{
    return on_host(ctx, batch, { in2 }, { out2 }, ModSwitch{ false, L, 2 });
}

int sb200_relinearize_sized(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *in, const sb200_kswitch_key *key,
                            uint64_t *out, void *stream)
{
    SB_NEED(key);
    return on_stream(ctx, stream, batch, { in }, { out }, RelinearizeSized{ L, size, key->k });
}
int sb200_relinearize_sized_host(sb200_context *ctx, size_t L, size_t size, size_t batch, const uint64_t *in, const sb200_kswitch_key *key,
                                 uint64_t *out)
{
    SB_NEED(key);
    return on_host(ctx, batch, { in }, { out }, RelinearizeSized{ L, size, key->k });
}

int sb200_apply_galois(sb200_context *ctx, size_t L, size_t batch, const uint64_t *in2, uint32_t elt, const sb200_kswitch_key *key,
                       uint64_t *out2, void *stream)
{
    SB_NEED(key);
    return on_stream(ctx, stream, batch, { in2 }, { out2 }, ApplyGalois{ L, elt, key->k });
}
int sb200_apply_galois_host(sb200_context *ctx, size_t L, size_t batch, const uint64_t *in2, uint32_t elt, const sb200_kswitch_key *key,
                            uint64_t *out2)
{
    SB_NEED(key);
    return on_host(ctx, batch, { in2 }, { out2 }, ApplyGalois{ L, elt, key->k });
}
int sb200_apply_galois_add(sb200_context *ctx, size_t L, size_t batch, const uint64_t *in2, uint32_t elt, const sb200_kswitch_key *key,
                           const uint64_t *addend2, uint64_t *out2, void *stream)
{
    SB_NEED(key);
    return on_stream(ctx, stream, batch, { in2, addend2 }, { out2 }, ApplyGaloisAdd{ L, elt, key->k });
}
int sb200_apply_galois_add_host(sb200_context *ctx, size_t L, size_t batch, const uint64_t *a, uint32_t elt, const sb200_kswitch_key *key,
                                const uint64_t *b, uint64_t *out2)
{
    SB_NEED(key);
    return on_host(ctx, batch, { a, b }, { out2 }, ApplyGaloisAdd{ L, elt, key->k });
}
int sb200_rotate_sum(sb200_context *ctx, size_t L, size_t batch, const uint64_t *in2, size_t steps, const uint32_t *elts,
                     const sb200_kswitch_key *const *keys, uint64_t *out2, void *stream)
{
    std::vector<const KSwitchKey *> k;
    if (int e = rotate_sum_keys(steps, elts, keys, k))
        return e;
    return on_stream(ctx, stream, batch, { in2 }, { out2 }, RotateSum{ L, steps, elts, k.data() });
}
int sb200_rotate_sum_host(sb200_context *ctx, size_t L, size_t batch, const uint64_t *in2, size_t steps, const uint32_t *elts,
                          const sb200_kswitch_key *const *keys, uint64_t *out2)
{
    std::vector<const KSwitchKey *> k;
    if (int e = rotate_sum_keys(steps, elts, keys, k))
        return e;
    return on_host(ctx, batch, { in2 }, { out2 }, RotateSum{ L, steps, elts, k.data() });
}
int sb200_apply_galois_multiply_plain_add(sb200_context *ctx, size_t L, size_t batch, const uint64_t *in2, uint32_t elt, const sb200_kswitch_key *key,
                                          size_t plain_count, const uint64_t *plain, const uint64_t *addend2, uint64_t *out2, void *stream)
{
    SB_NEED(key);
    return on_stream(ctx, stream, batch, { in2, plain, addend2 }, { out2 }, ApplyGaloisMultiplyPlainAdd{ L, plain_count, elt, key->k });
}
int sb200_apply_galois_multiply_plain_add_host(sb200_context *ctx, size_t L, size_t batch, const uint64_t *in2, uint32_t elt,
                                               const sb200_kswitch_key *key, size_t plain_count, const uint64_t *plain, const uint64_t *addend2,
                                               uint64_t *out2)
{
    SB_NEED(key);
    return on_host(ctx, batch, { in2, plain, addend2 }, { out2 }, ApplyGaloisMultiplyPlainAdd{ L, plain_count, elt, key->k });
}
int sb200_diagonal_sum(sb200_context *ctx, size_t L, size_t batch, const uint64_t *in2, size_t count, const uint32_t *elts,
                       const sb200_kswitch_key *const *keys, const size_t *plain_counts, const uint64_t *const *plains, int plain_is_ntt,
                       uint64_t *out2, void *stream)
{
    std::vector<const KSwitchKey *> k;
    if (int e = diagonal_sum_keys(count, elts, keys, plain_counts, plains, k))
        return e;
    return on_stream(ctx, stream, batch, InSlabs(&in2, 1, plains, count), { out2 },
                     DiagonalSum{ L, count, elts, k.data(), plain_counts, plain_is_ntt != 0 });
}
int sb200_diagonal_sum_host(sb200_context *ctx, size_t L, size_t batch, const uint64_t *in2, size_t count, const uint32_t *elts,
                            const sb200_kswitch_key *const *keys, const size_t *plain_counts, const uint64_t *const *plains, int plain_is_ntt,
                            uint64_t *out2)
{
    std::vector<const KSwitchKey *> k;
    if (int e = diagonal_sum_keys(count, elts, keys, plain_counts, plains, k))
        return e;
    return on_host(ctx, batch, InSlabs(&in2, 1, plains, count), { out2 }, DiagonalSum{ L, count, elts, k.data(), plain_counts, plain_is_ntt != 0 });
}

// ---- wire format (SURVEY 8f rank 3): Ciphertext::save / load, compr_mode none, between byte streams and device slabs ----
int sb200_get_parms_id(const sb200_context *ctx, size_t L, uint64_t out[4])
{
    SB_NEED(ctx);
    SB_NEED(out);
    SB_TRY
    const Context &c = *ctx->c;
    if (L < 1 || L > c.k)
        throw std::out_of_range("L");
    for (int i = 0; i < 4; i++)
        out[i] = c.parms_ids[L - 1][i];
    return SB200_OK;
    SB_CATCH
}

int sb200_ciphertext_inspect(const uint8_t *stream, size_t len, sb200_ct_info *info)
{
    SB_NEED(stream);
    SB_NEED(info);
    SB_TRY
    std::vector<uint8_t> plain;
    // a compressed object is inflated first (bounded by the largest ciphertext the format allows: 16 x 256 x 131072 words)
    if (sbw::inflate_stream(stream, len, sbw::save_size(size_t(16) * 256 * 131072) + 128, plain))
    {
        sbw::inspect(plain.data(), plain.size(), *info);
        uint64_t total = 0;
        std::memcpy(&total, stream + 8, sizeof(total)); // SEALHeader::size of the stream as given
        info->stream_bytes = total;
        info->compr_mode = 1;
    }
    else
        sbw::inspect(stream, len, *info);
    return SB200_OK;
    SB_CATCH
}

size_t sb200_ciphertext_save_size(const sb200_context *ctx, size_t L, size_t size)
{
    return ctx ? sbw::save_size(size * L * ctx->c->n) : 0;
}

int sb200_ciphertext_load(sb200_context *ctx, size_t batch, const uint8_t *const *streams, const size_t *lens, size_t L, size_t size,
                          int validate, uint64_t *d_out, sb200_ct_info *infos, void *stream)
{
    SB_NEED(streams);
    SB_NEED(lens);
    SB_NEED(d_out);
    SB_TRY
    SB_ENTER_STREAM(ctx, stream)
    check_level(c, L, batch);
    auto st = static_cast<cudaStream_t>(stream);
    const size_t words = size * L * c.n;
    // seeded members, blake2xb ones first so that each PRNG type is one launch: 8 words of seed each, the prng_type, and the word
    // offset of their second polynomial in d_out
    std::vector<u64> seeds[2];
    std::vector<int> types[2];
    std::vector<long long> seed_dst[2];
    for (size_t b = 0; b < batch; b++)
    {
        sb200_ct_info info;
        std::vector<uint8_t> plain; // a zlib-compressed member is inflated on the host (bounded by the shape asked for)
        const uint8_t *src = streams[b];
        if (!src)
            throw std::invalid_argument("in cannot be null");
        if (sbw::inflate_stream(src, lens[b], sbw::save_size(words) + 128, plain))
        {
            sbw::inspect(plain.data(), plain.size(), info);
            src = plain.data();
            info.compr_mode = 1;
        }
        else
            sbw::inspect(src, lens[b], info);
        // is_metadata_valid_for (ciphertext.cpp:299-302): the stream must belong to this context at the level asked for
        if (info.poly_modulus_degree != c.n || info.coeff_modulus_size != L || info.size != size ||
            std::memcmp(info.parms_id, c.parms_ids[L - 1].data(), sizeof(info.parms_id)) != 0)
            throw std::logic_error("ciphertext data is invalid");
        if (infos)
            infos[b] = info;
        // (pageable source: the call returns once the bytes have left the buffer, so `plain` may go out of scope)
        cuda_check(cudaMemcpyAsync(d_out + b * words, src + info.data_offset, info.data_words * sizeof(u64), cudaMemcpyHostToDevice, st), "H2D");
        if (info.seeded) // UniformRandomGeneratorInfo::make_prng: the stream names its PRNG (randomgen.cpp:163-177)
        {
            const int t = info.seeded == kPrngShake256;
            u64 sd[8];
            std::memcpy(sd, src + info.seed_offset, sizeof(sd));
            seeds[t].insert(seeds[t].end(), sd, sd + 8);
            types[t].push_back(info.seeded);
            seed_dst[t].push_back(static_cast<long long>(b * words + L * c.n));
        }
    }
    seeds[0].insert(seeds[0].end(), seeds[1].begin(), seeds[1].end());
    types[0].insert(types[0].end(), types[1].begin(), types[1].end());
    seed_dst[0].insert(seed_dst[0].end(), seed_dst[1].begin(), seed_dst[1].end());
    if (!seed_dst[0].empty()) // Ciphertext::expand_seed
        op_expand_seeded(c, L, seed_dst[0].size(), seeds[0].data(), types[0].data(), seed_dst[0].data(), reinterpret_cast<u64 *>(d_out), st);
    if (validate && !op_residues_in_range(c, L, batch * size * L, reinterpret_cast<const u64 *>(d_out), st))
        throw std::logic_error("ciphertext data is invalid"); // Ciphertext::load -> is_valid_for (ciphertext.h:640-655)
    return SB200_OK;
    SB_CATCH
}

int sb200_ciphertext_save(sb200_context *ctx, size_t batch, size_t L, size_t size, const uint64_t *d_in, const sb200_ct_info *meta,
                          uint8_t *const *outs, size_t capacity, void *stream)
{
    SB_NEED(d_in);
    SB_NEED(meta);
    SB_NEED(outs);
    SB_TRY
    SB_ENTER_STREAM(ctx, stream)
    check_level(c, L, batch);
    auto st = static_cast<cudaStream_t>(stream);
    const size_t words = size * L * c.n;
    if (size < 2 || size > 16)
        throw std::invalid_argument("invalid size");
    if (capacity < sbw::save_size(words))
        throw std::invalid_argument("insufficient size"); // Serialization::Save into a too small buffer
    for (size_t b = 0; b < batch; b++)
    {
        if (!outs[b])
            throw std::invalid_argument("out cannot be null");
        sb200_ct_info info = meta[b];
        std::memcpy(info.parms_id, c.parms_ids[L - 1].data(), sizeof(info.parms_id));
        info.size = size, info.poly_modulus_degree = c.n, info.coeff_modulus_size = L, info.data_words = words;
        sbw::write_prefix(info, outs[b]);
        cuda_check(cudaMemcpyAsync(outs[b] + sbw::kDataOffset, d_in + b * words, words * sizeof(u64), cudaMemcpyDeviceToHost, st), "D2H");
    }
    cuda_check(cudaStreamSynchronize(st), "synchronize");
    return SB200_OK;
    SB_CATCH
}

// ---- decryption (SURVEY 8f rank 4): Decryptor(context, secret_key) + Decryptor::decrypt ----
int sb200_secret_key_create(sb200_context *ctx, const uint64_t *h_secret_key, sb200_secret_key **out)
{
    SB_NEED(h_secret_key);
    SB_NEED(out);
    SB_TRY
    SB_ENTER(ctx)
    auto h = std::make_unique<sb200_secret_key>();
    secret_key_create(c, (const u64 *)h_secret_key, h->k);
    *out = h.release();
    return SB200_OK;
    SB_CATCH
}

int sb200_secret_key_destroy(sb200_secret_key *key)
{
    SB_NEED(key);
    delete key;
    return SB200_OK;
}

// ---- Encryptor(context, public_key)::encrypt_zero (sb_prng.cu) ----
int sb200_public_key_create(sb200_context *ctx, const uint64_t *h_public_key, sb200_public_key **out)
{
    SB_NEED(h_public_key);
    SB_NEED(out);
    SB_TRY
    SB_ENTER(ctx)
    auto h = std::make_unique<sb200_public_key>();
    public_key_create(c, (const u64 *)h_public_key, h->k);
    *out = h.release();
    return SB200_OK;
    SB_CATCH
}

int sb200_public_key_destroy(sb200_public_key *key)
{
    SB_NEED(key);
    delete key;
    return SB200_OK;
}

namespace
{
    // fresh PRNG seeds from the OS entropy source, as UniformRandomGeneratorFactory::create does (randomgen.cpp:34-50); wiped on scope exit
    struct FreshSeeds
    {
        std::vector<u64> words;
        explicit FreshSeeds(size_t batch) : words(batch * 8)
        {
            std::random_device rd("/dev/urandom");
            for (auto &w : words)
                w = (static_cast<u64>(rd()) << 32) | static_cast<u64>(rd());
        }
        ~FreshSeeds()
        {
            volatile u64 *w = words.data(); // the seeds determine the noise: do not leave them on the heap
            for (size_t i = 0; i < words.size(); i++)
                w[i] = 0;
        }
    };
} // namespace

int sb200_encrypt_zero_asymmetric(sb200_context *ctx, sb200_public_key *key, size_t L, size_t batch, const uint64_t *h_seeds, uint64_t *d_out,
                                  void *stream)
{
    return sb200_encrypt_zero_asymmetric_prng(ctx, key, L, batch, kPrngBlake2xb, h_seeds, d_out, stream);
}

int sb200_encrypt_zero_asymmetric_prng(sb200_context *ctx, sb200_public_key *key, size_t L, size_t batch, int prng, const uint64_t *h_seeds,
                                       uint64_t *d_out, void *stream)
{
    SB_NEED(key);
    SB_NEED(d_out);
    SB_TRY
    SB_ENTER_STREAM(ctx, stream)
    check_level(c, L, batch);
    std::unique_ptr<FreshSeeds> fresh;
    if (!h_seeds)
    {
        fresh = std::make_unique<FreshSeeds>(batch);
        h_seeds = reinterpret_cast<const uint64_t *>(fresh->words.data());
    }
    // returns after a stream synchronisation: the seeds may be wiped
    check_prng_type(prng);
    op_encrypt_zero_asymmetric(c, key->k, L, batch, (const u64 *)h_seeds, prng, (u64 *)d_out, static_cast<cudaStream_t>(stream));
    return SB200_OK;
    SB_CATCH
}

int sb200_encrypt_asymmetric(sb200_context *ctx, sb200_public_key *key, size_t L, size_t batch, const uint64_t *d_plain, int prng,
                             const uint64_t *h_seeds, uint64_t *d_out, void *stream)
{
    SB_NEED(key);
    SB_NEED(d_plain);
    SB_NEED(d_out);
    SB_TRY
    SB_ENTER_STREAM(ctx, stream)
    check_level(c, L, batch);
    if (d_plain == d_out)
        throw std::invalid_argument("d_plain must not alias d_out");
    check_prng_type(prng);
    std::unique_ptr<FreshSeeds> fresh;
    if (!h_seeds)
    {
        fresh = std::make_unique<FreshSeeds>(batch);
        h_seeds = reinterpret_cast<const uint64_t *>(fresh->words.data());
    }
    op_encrypt_asymmetric(c, key->k, L, batch, (const u64 *)d_plain, (const u64 *)h_seeds, prng, (u64 *)d_out, static_cast<cudaStream_t>(stream));
    return SB200_OK;
    SB_CATCH
}

// ---- CKKSEncoder::encode / decode (sb_ckks.cu) ----
int sb200_ckks_encode(sb200_context *ctx, size_t L, size_t batch, const double *d_values, size_t count, int is_complex, double scale,
                      uint64_t *d_plain, void *stream)
{
    return on_stream(ctx, stream, batch, { d_values }, { d_plain }, CkksEncode{ L, count, is_complex != 0, d_values != nullptr, scale });
}
int sb200_ckks_encode_host(sb200_context *ctx, size_t L, size_t batch, const double *h_values, size_t count, int is_complex, double scale,
                           uint64_t *h_plain)
{
    return on_host(ctx, batch, { h_values }, { h_plain }, CkksEncode{ L, count, is_complex != 0, h_values != nullptr, scale });
}

int sb200_ckks_encode_scalar(sb200_context *ctx, size_t L, size_t batch, int kind, const void *d_values, double scale, uint64_t *d_plain,
                             void *stream)
{
    return on_stream(ctx, stream, batch, { d_values }, { d_plain }, CkksEncodeScalar{ L, kind, scale, nullptr });
}
int sb200_ckks_encode_scalar_host(sb200_context *ctx, size_t L, size_t batch, int kind, const void *h_values, double scale,
                                  uint64_t *h_plain)
{
    return on_host(ctx, batch, { h_values }, { h_plain }, CkksEncodeScalar{ L, kind, scale, static_cast<const u64 *>(h_values) });
}

int sb200_ckks_decode(sb200_context *ctx, size_t L, size_t batch, const uint64_t *d_plain, double scale, double *d_values, void *stream)
{
    return on_stream(ctx, stream, batch, { d_plain }, { d_values }, CkksDecode{ L, scale });
}
int sb200_ckks_decode_host(sb200_context *ctx, size_t L, size_t batch, const uint64_t *h_plain, double scale, double *h_values)
{
    return on_host(ctx, batch, { h_plain }, { h_values }, CkksDecode{ L, scale });
}

// Encryptor::encrypt_zero_symmetric for a batch (sb_prng.cu); h_bootstrap_seeds == nullptr: fresh seeds from the OS entropy source,
// as UniformRandomGeneratorFactory::create does through random_uint64 (randomgen.cpp:34-50)
int sb200_encrypt_zero_symmetric(sb200_context *ctx, sb200_secret_key *key, size_t L, size_t batch, const uint64_t *h_bootstrap_seeds,
                                 int save_seed, uint64_t *d_out, uint64_t *h_public_seeds, void *stream)
{
    return sb200_encrypt_zero_symmetric_prng(ctx, key, L, batch, kPrngBlake2xb, kPrngBlake2xb, h_bootstrap_seeds, save_seed, d_out, h_public_seeds,
                                             stream);
}

int sb200_encrypt_zero_symmetric_prng(sb200_context *ctx, sb200_secret_key *key, size_t L, size_t batch, int bootstrap_prng, int ciphertext_prng,
                                      const uint64_t *h_bootstrap_seeds, int save_seed, uint64_t *d_out, uint64_t *h_public_seeds, void *stream)
{
    SB_NEED(key);
    SB_NEED(d_out);
    SB_TRY
    SB_ENTER_STREAM(ctx, stream)
    check_level(c, L, batch);
    std::unique_ptr<FreshSeeds> fresh;
    if (!h_bootstrap_seeds)
    {
        fresh = std::make_unique<FreshSeeds>(batch);
        h_bootstrap_seeds = reinterpret_cast<const uint64_t *>(fresh->words.data());
    }
    check_prng_type(bootstrap_prng);
    check_prng_type(ciphertext_prng);
    op_encrypt_zero_symmetric(c, key->k, L, batch, (const u64 *)h_bootstrap_seeds, bootstrap_prng, ciphertext_prng, save_seed != 0, (u64 *)d_out,
                              (u64 *)h_public_seeds, static_cast<cudaStream_t>(stream));
    // op_encrypt_zero_symmetric synchronised the stream while expanding c_1: the seeds have been consumed and may be wiped
    return SB200_OK;
    SB_CATCH
}

int sb200_encrypt_symmetric(sb200_context *ctx, sb200_secret_key *key, size_t L, size_t batch, const uint64_t *d_plain, int bootstrap_prng,
                            int ciphertext_prng, const uint64_t *h_bootstrap_seeds, int save_seed, uint64_t *d_out, uint64_t *h_public_seeds,
                            void *stream)
{
    SB_NEED(key);
    SB_NEED(d_plain);
    SB_NEED(d_out);
    SB_TRY
    SB_ENTER_STREAM(ctx, stream)
    check_level(c, L, batch);
    if (d_plain == d_out)
        throw std::invalid_argument("d_plain must not alias d_out");
    check_prng_type(bootstrap_prng);
    check_prng_type(ciphertext_prng);
    std::unique_ptr<FreshSeeds> fresh;
    if (!h_bootstrap_seeds)
    {
        fresh = std::make_unique<FreshSeeds>(batch);
        h_bootstrap_seeds = reinterpret_cast<const uint64_t *>(fresh->words.data());
    }
    op_encrypt_symmetric(c, key->k, L, batch, (const u64 *)d_plain, (const u64 *)h_bootstrap_seeds, bootstrap_prng, ciphertext_prng, save_seed != 0,
                         (u64 *)d_out, (u64 *)h_public_seeds, static_cast<cudaStream_t>(stream));
    // as above: the stream was synchronised while c_1 was expanded
    return SB200_OK;
    SB_CATCH
}

// ---- KeyGenerator(context, secret_key)::create_public_key / create_relin_keys / create_galois_keys (sb_prng.cu) ----
// The key is generated into the storage of the handle it becomes; when only the host words are asked for, that handle is a
// temporary that goes away after the download.
int sb200_public_key_generate(sb200_context *ctx, sb200_secret_key *key, int bootstrap_prng, int ciphertext_prng, const uint64_t *h_bootstrap_seed,
                              uint64_t *h_public_key, sb200_public_key **out)
{
    SB_NEED(key);
    if (!h_public_key && !out)
    {
        g_last_error = "null pointer: h_public_key and out";
        return SB200_E_POINTER;
    }
    SB_TRY
    SB_ENTER_STREAM(ctx, nullptr)
    std::unique_ptr<FreshSeeds> fresh;
    if (!h_bootstrap_seed)
    {
        fresh = std::make_unique<FreshSeeds>(1);
        h_bootstrap_seed = reinterpret_cast<const uint64_t *>(fresh->words.data());
    }
    auto h = std::make_unique<sb200_public_key>();
    h->k.d_key = DevBuf<u64>(2 * c.k * c.n);
    h->k.ctx = &c;
    const size_t bytes = h->k.d_key.bytes();
    op_generate_public_key(c, key->k, bootstrap_prng, ciphertext_prng, (const u64 *)h_bootstrap_seed, h->k.d_key.get(), nullptr);
    cuda_check(cudaStreamSynchronize(nullptr), "synchronize");
    if (h_public_key)
        cuda_check(cudaMemcpy(h_public_key, h->k.d_key.get(), bytes, cudaMemcpyDeviceToHost), "download public key");
    if (out)
        *out = h.release();
    return SB200_OK;
    SB_CATCH
}

int sb200_kswitch_key_generate(sb200_context *ctx, sb200_secret_key *key, uint32_t galois_elt, int bootstrap_prng, int ciphertext_prng,
                               const uint64_t *h_bootstrap_seeds, uint64_t *h_key, sb200_kswitch_key **out)
{
    SB_NEED(key);
    if (!h_key && !out)
    {
        g_last_error = "null pointer: h_key and out";
        return SB200_E_POINTER;
    }
    SB_TRY
    SB_ENTER_STREAM(ctx, nullptr)
    const size_t digits = std::max<size_t>(c.k, 2) - 1; // k < 2 is rejected by op_generate_kswitch_key
    std::unique_ptr<FreshSeeds> fresh;
    if (!h_bootstrap_seeds)
    {
        fresh = std::make_unique<FreshSeeds>(digits);
        h_bootstrap_seeds = reinterpret_cast<const uint64_t *>(fresh->words.data());
    }
    auto h = kswitch_key_alloc(c, digits);
    op_generate_kswitch_key(c, key->k, galois_elt, bootstrap_prng, ciphertext_prng, (const u64 *)h_bootstrap_seeds, h->k.d_key.get(), nullptr);
    cuda_check(cudaStreamSynchronize(nullptr), "synchronize");
    if (h_key)
        cuda_check(cudaMemcpy(h_key, h->k.d_key.get(), digits * 2 * c.k * c.n * sizeof(u64), cudaMemcpyDeviceToHost), "download key");
    if (out)
    {
        if (!kswitch_key_finish(c, h->k))
            throw std::logic_error("kswitch key data is not valid for encryption parameters");
        *out = h.release();
    }
    return SB200_OK;
    SB_CATCH
}

} // extern "C"

// ---- seed-compressed output: Serializable<Ciphertext> / <PublicKey> / <RelinKeys> / <GaloisKeys>::save(compr_mode_type::none) ----
namespace
{
    // the metadata of a key-level member of a key (util/rlwe.cpp:282-287 with is_ntt_form = true): NTT form, scale 1, correction factor 1
    sb200_ct_info key_member_info(const Context &c)
    {
        sb200_ct_info info{};
        std::memcpy(info.parms_id, c.parms_ids[c.k - 1].data(), sizeof(info.parms_id));
        info.size = 2, info.poly_modulus_degree = c.n, info.coeff_modulus_size = c.k, info.data_words = c.k * c.n;
        info.is_ntt_form = 1, info.scale = 1.0, info.correction_factor = 1;
        return info;
    }

    // The keys of one seeded RelinKeys / GaloisKeys stream.  {0} is create_relin_keys (one slot); otherwise create_galois_keys: the
    // elements in the order given with duplicates skipped (GaloisKeys::has_key, keygenerator.cpp:190-205), in n slots.
    struct KeySet
    {
        std::vector<uint32_t> elts;  // distinct elements in draw order
        size_t slots = 0;
        std::vector<size_t> filled;  // their slot indices, ascending
        size_t slot_of(uint32_t elt) const { return slots == 1 ? 0 : (elt - 1) / 2; }
    };
    KeySet key_set(const Context &c, const uint32_t *elts, size_t count)
    {
        KeySet s;
        const bool relin = count == 1 && elts[0] == 0;
        s.slots = relin ? 1 : c.n;
        for (size_t i = 0; i < count; i++)
        {
            const uint32_t e = elts[i];
            if (!relin && e == 0)
                throw std::invalid_argument("galois_elts: 0 (relinearization) cannot be mixed with Galois elements");
            if (!relin && (!(e & 1) || e >= 2 * c.n))
                throw std::invalid_argument("Galois element is not valid"); // keygenerator.cpp:195-199
            if (std::find(s.elts.begin(), s.elts.end(), e) == s.elts.end())
                s.elts.push_back(e);
        }
        for (const uint32_t e : s.elts)
            s.filled.push_back(s.slot_of(e));
        std::sort(s.filled.begin(), s.filled.end());
        return s;
    }
    size_t kswitch_stream_bytes(const Context &c, const KeySet &s)
    {
        return sbw::kswitch_save_size(s.slots, s.elts.size(), c.k - 1, sbw::seeded_save_size(c.k * c.n));
    }

    // one staged download in flight on a helper thread while the calling thread generates the next chunk
    struct PendingCopy
    {
        std::thread t;
        std::exception_ptr err;
        void wait()
        {
            if (t.joinable())
                t.join();
            if (err)
            {
                std::exception_ptr e = err;
                err = nullptr;
                std::rethrow_exception(e);
            }
        }
        ~PendingCopy()
        {
            if (t.joinable())
                t.join();
        }
    };
} // namespace

extern "C" {
size_t sb200_ciphertext_save_seeded_size(const sb200_context *ctx, size_t L)
{
    return ctx ? sbw::seeded_save_size(L * ctx->c->n) : 0;
}

int sb200_ciphertext_save_seeded(sb200_context *ctx, size_t batch, size_t L, const uint64_t *d_in, const sb200_ct_info *meta,
                                 const uint64_t *h_public_seeds, int prng, uint8_t *const *outs, size_t capacity, void *stream)
{
    SB_NEED(d_in);
    SB_NEED(meta);
    SB_NEED(h_public_seeds);
    SB_NEED(outs);
    SB_TRY
    SB_ENTER_STREAM(ctx, stream)
    check_level(c, L, batch);
    check_prng_type(prng);
    auto st = static_cast<cudaStream_t>(stream);
    const size_t words = L * c.n; // c_0
    if (capacity < sbw::seeded_save_size(words))
        throw std::invalid_argument("insufficient size"); // Serialization::Save into a too small buffer
    for (size_t b = 0; b < batch; b++)
        if (!outs[b])
            throw std::invalid_argument("out cannot be null");
    for (size_t b = 0; b < batch; b++)
    {
        sb200_ct_info info = meta[b];
        std::memcpy(info.parms_id, c.parms_ids[L - 1].data(), sizeof(info.parms_id));
        info.size = 2, info.poly_modulus_degree = c.n, info.coeff_modulus_size = L, info.data_words = words;
        sbw::write_seeded(info, prng, reinterpret_cast<const u64 *>(h_public_seeds) + b * 8, outs[b]);
        cuda_check(cudaMemcpyAsync(outs[b] + sbw::kDataOffset, d_in + b * 2 * words, words * sizeof(u64), cudaMemcpyDeviceToHost, st), "D2H");
    }
    cuda_check(cudaStreamSynchronize(st), "synchronize");
    return SB200_OK;
    SB_CATCH
}

int sb200_public_key_generate_seeded(sb200_context *ctx, sb200_secret_key *key, int bootstrap_prng, int ciphertext_prng,
                                     const uint64_t *h_bootstrap_seed, uint8_t *out, size_t capacity, sb200_public_key **handle)
{
    SB_NEED(key);
    SB_NEED(out);
    SB_TRY
    SB_ENTER_STREAM(ctx, nullptr)
    check_prng_type(bootstrap_prng);
    check_prng_type(ciphertext_prng);
    if (!key->k.d_pow || key->k.ctx != &c)
        throw std::invalid_argument("secret key is not valid for encryption parameters");
    const sb200_ct_info info = key_member_info(c);
    if (capacity < sbw::seeded_save_size(info.data_words))
        throw std::invalid_argument("insufficient size");
    std::unique_ptr<FreshSeeds> fresh;
    if (!h_bootstrap_seed)
    {
        fresh = std::make_unique<FreshSeeds>(1);
        h_bootstrap_seed = reinterpret_cast<const uint64_t *>(fresh->words.data());
    }
    auto h = std::make_unique<sb200_public_key>();
    h->k.d_key = DevBuf<u64>(2 * c.k * c.n);
    h->k.ctx = &c;
    u64 pub[8];
    op_generate_public_key(c, key->k, bootstrap_prng, ciphertext_prng, (const u64 *)h_bootstrap_seed, h->k.d_key.get(), nullptr, pub);
    sbw::write_seeded(info, ciphertext_prng, pub, out);
    cuda_check(cudaMemcpy(out + sbw::kDataOffset, h->k.d_key.get(), info.data_words * sizeof(u64), cudaMemcpyDeviceToHost), "download c_0");
    if (handle)
        *handle = h.release();
    return SB200_OK;
    SB_CATCH
}

size_t sb200_kswitch_keys_save_seeded_size(const sb200_context *ctx, const uint32_t *galois_elts, size_t count)
{
    if (!ctx || !galois_elts || ctx->c->k < 2)
        return 0;
    try
    {
        return kswitch_stream_bytes(*ctx->c, key_set(*ctx->c, galois_elts, count));
    }
    catch (const std::exception &e)
    {
        g_last_error = e.what();
        return 0;
    }
}

// Each key's digits are generated into one of two device buffers (alternating by key, so that the download of one key's last chunk
// overlaps the generation of the next key's first); after each chunk, the seed infos are written and the chunk's c_0 rows go to
// their members through the context's page-locked download lane on a helper thread while the next chunk is generated.
int sb200_kswitch_keys_generate_seeded(sb200_context *ctx, sb200_secret_key *key, const uint32_t *galois_elts, size_t count, int bootstrap_prng,
                                       int ciphertext_prng, const uint64_t *h_bootstrap_seeds, uint8_t *out, size_t capacity)
{
    SB_NEED(key);
    SB_NEED(galois_elts);
    SB_NEED(out);
    SB_TRY
    SB_ENTER_STREAM(ctx, nullptr)
    if (c.k < 2)
        throw std::logic_error("keyswitching is not supported by the context"); // keygenerator.cpp:329-332
    const KeySet ks = key_set(c, galois_elts, count);
    check_prng_type(bootstrap_prng);
    check_prng_type(ciphertext_prng);
    if (!key->k.d_pow || key->k.ctx != &c)
        throw std::invalid_argument("secret key is not valid for encryption parameters");
    if (capacity < kswitch_stream_bytes(c, ks))
        throw std::invalid_argument("insufficient size");
    const size_t digits = c.k - 1, poly = c.k * c.n, E = ks.elts.size();
    const sb200_ct_info info = key_member_info(c);
    const size_t member = sbw::seeded_save_size(info.data_words);
    std::unique_ptr<FreshSeeds> fresh;
    if (!h_bootstrap_seeds)
    {
        fresh = std::make_unique<FreshSeeds>(E * digits);
        h_bootstrap_seeds = reinterpret_cast<const uint64_t *>(fresh->words.data());
    }
    std::vector<size_t> first;
    sbw::write_kswitch_frame(reinterpret_cast<const u64 *>(info.parms_id), ks.slots, ks.filled, digits, member, out, first);
    DevBuf<u64> buf[2];
    buf[0] = DevBuf<u64>(digits * 2 * poly);
    if (E > 1)
        buf[1] = DevBuf<u64>(digits * 2 * poly);
    std::vector<u64> pub(digits * 8); // public seeds: what the stream carries
    std::vector<uint64_t *> rows(digits);
    PendingCopy pending; // declared last: joined before the buffers above go away
    for (size_t e = 0; e < E; e++)
    {
        const size_t f = static_cast<size_t>(std::lower_bound(ks.filled.begin(), ks.filled.end(), ks.slot_of(ks.elts[e])) - ks.filled.begin());
        uint8_t *slot = out + first[f];
        u64 *d = buf[e & 1].get();
        op_generate_kswitch_key(c, key->k, ks.elts[e], bootstrap_prng, ciphertext_prng, (const u64 *)h_bootstrap_seeds + e * digits * 8, d, nullptr,
                                pub.data(), [&](size_t d0, size_t cnt) {
                                    pending.wait();
                                    for (size_t j = d0; j < d0 + cnt; j++)
                                    {
                                        sbw::write_seeded(info, ciphertext_prng, pub.data() + j * 8, slot + j * member);
                                        rows[j] = reinterpret_cast<uint64_t *>(slot + j * member + sbw::kDataOffset);
                                    }
                                    // the chunk is complete (op_generate_kswitch_key synchronised): no wait on the default stream
                                    pending.t = std::thread([&c, &pending, &rows, d, d0, cnt, poly] {
                                        try
                                        {
                                            rows_transfer(c, false, reinterpret_cast<uint64_t *>(d + d0 * 2 * poly), rows.data() + d0, poly * sizeof(u64), cnt,
                                                          2 * poly * sizeof(u64), false);
                                        }
                                        catch (...)
                                        {
                                            pending.err = std::current_exception();
                                        }
                                    });
                                });
    }
    pending.wait();
    return SB200_OK;
    SB_CATCH
}
} // extern "C"

// the decryption phases and plaintexts do not stay behind in the arenas (the reference decrypts inside a clear-on-destruction pool,
// decryptor.cpp:106-109)
namespace
{
    void wipe_stream(Context &c, cudaStream_t st) { c.wipe_scratch(st); }
    void wipe_host(Context &c, cudaStream_t st)
    {
        c.wipe_scratch(st);
        for (int slot = 0; slot < 2; slot++) // and the output staging
            if (c.io.buf[slot][2])
                cuda_check(cudaMemsetAsync(c.io.buf[slot][2].get(), 0, c.io.buf[slot][2].bytes(), st), "wipe staging");
        cuda_check(cudaStreamSynchronize(st), "synchronize");
    }
} // namespace

extern "C" {
int sb200_decrypt(sb200_context *ctx, sb200_secret_key *key, size_t L, size_t size, size_t batch, const uint64_t *ct,
                  const uint64_t *h_correction_factors, uint64_t *plain, void *stream)
{
    SB_NEED(key);
    return on_stream(ctx, stream, batch, { ct }, { plain }, Decrypt{ key->k, L, size, (const u64 *)h_correction_factors }, wipe_stream);
}

int sb200_decrypt_host(sb200_context *ctx, sb200_secret_key *key, size_t L, size_t size, size_t batch, const uint64_t *ct,
                       const uint64_t *h_correction_factors, uint64_t *plain)
{
    SB_NEED(key);
    return on_host(ctx, batch, { ct }, { plain }, Decrypt{ key->k, L, size, (const u64 *)h_correction_factors }, wipe_host);
}

// Decryptor::invariant_noise_budget: the phases depend on the secret key, so the arenas are wiped as after a decryption
int sb200_invariant_noise_budget(sb200_context *ctx, sb200_secret_key *key, size_t L, size_t size, size_t batch, const uint64_t *d_ct,
                                 int *d_budgets, void *stream)
{
    SB_NEED(key);
    return on_stream(ctx, stream, batch, { d_ct }, { d_budgets }, NoiseBudget{ key->k, L, size }, wipe_stream);
}

int sb200_invariant_noise_budget_host(sb200_context *ctx, sb200_secret_key *key, size_t L, size_t size, size_t batch, const uint64_t *h_ct,
                                      int *h_budgets)
{
    SB_NEED(key);
    return on_host(ctx, batch, { h_ct }, { h_budgets }, NoiseBudget{ key->k, L, size }, wipe_host);
}

} // extern "C"
