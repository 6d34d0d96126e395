/* DLPack through the C++ interface: CUDAArray<T>::to_dlpack / from_dlpack (include/enoki/cuda.h).
 *   - a CUDAArray<float> (legacy tensor) and a CUDAArray<uint8_t> (versioned tensor) are exported and imported back:
 *     both directions alias the same buffer and the values survive;
 *   - a tensor of the wrong dtype is refused and stays the caller's;
 *   - a hand-built 2-D DLManagedTensor over cudaMalloc memory is imported, feeds an evaluation, and its deleter has
 *     run exactly once after cuda_sync().
 * Prints "dlpack_check ok". */
#include <enoki/cuda.h>
#include <cuda_runtime.h>
#include <cstdio>
#include <vector>

using namespace enoki;
using FloatC = CUDAArray<float>;
using UInt8C = CUDAArray<uint8_t>;

#define CHECK(cond)                                                                    \
    do {                                                                               \
        if (!(cond)) {                                                                 \
            fprintf(stderr, "dlpack_check: %s failed (line %d)\n", #cond, __LINE__);   \
            return 1;                                                                  \
        }                                                                              \
    } while (0)

static int g_deleted = 0;

static void counting_deleter(DLManagedTensor *self) {
    ++g_deleted;
    cudaFree(self->dl_tensor.data);
    delete[] self->dl_tensor.shape;
    delete self;
}

template <typename T> static std::vector<T> host(const CUDAArray<T> &a) {
    a.eval();
    std::vector<T> out(a.size());
    ek_memcpy_from_device(out.data(), a.data(), out.size() * sizeof(T));
    return out;
}

int main() {
    cuda_init();
    const size_t n = 4097;
    std::vector<float> xf(n);
    std::vector<uint8_t> xu(n);
    for (size_t i = 0; i < n; ++i) { xf[i] = 0.25f * (float) i - 100.f; xu[i] = (uint8_t) (i * 7); }

    {   /* float: legacy tensor, export -> import */
        FloatC a = FloatC::copy(xf.data(), n);
        a.eval();
        DLManagedTensor *m = a.to_dlpack();
        CHECK(m->dl_tensor.data == a.data() && m->dl_tensor.ndim == 1 && m->dl_tensor.shape[0] == (int64_t) n);
        CHECK(m->dl_tensor.dtype.code == kDLFloat && m->dl_tensor.dtype.bits == 32 && m->dl_tensor.dtype.lanes == 1);
        CHECK(m->dl_tensor.device.device_type == kDLCUDA && m->dl_tensor.device.device_id == ek_device());
        CHECK(m->dl_tensor.strides == nullptr && m->dl_tensor.byte_offset == 0);
        bool refused = false;
        try { (void) UInt8C::from_dlpack(m); } catch (const std::runtime_error &) { refused = true; }
        CHECK(refused);                                   /* ... and m is still ours */
        FloatC b = FloatC::from_dlpack(m);
        CHECK(b.data() == a.data() && b.size() == n);
        CHECK(host(b) == xf);
        std::vector<float> twice = host(FloatC(b * 2.f));
        for (size_t i = 0; i < n; ++i) CHECK(twice[i] == xf[i] * 2.f);
    }
    {   /* uint8: versioned tensor, export -> import */
        UInt8C a = UInt8C::copy(xu.data(), n);
        a.eval();
        DLManagedTensorVersioned *m = a.to_dlpack_versioned();
        CHECK(m->version.major == 1 && m->flags == 0);
        CHECK(m->dl_tensor.dtype.code == kDLUInt && m->dl_tensor.dtype.bits == 8);
        UInt8C b = UInt8C::from_dlpack(m);
        CHECK(b.data() == a.data());
        CHECK(host(b) == xu);
    }
    {   /* a foreign 10 x (n / 10) tensor with a counting deleter */
        const int64_t rows = 10, cols = (int64_t) n / 10, count = rows * cols;
        float *dev = nullptr;
        CHECK(cudaMalloc(&dev, count * sizeof(float)) == cudaSuccess);
        CHECK(cudaMemcpy(dev, xf.data(), count * sizeof(float), cudaMemcpyHostToDevice) == cudaSuccess);
        DLManagedTensor *m = new DLManagedTensor();
        m->dl_tensor.data = dev;
        m->dl_tensor.device = { kDLCUDA, ek_device() };
        m->dl_tensor.ndim = 2;
        m->dl_tensor.dtype = { kDLFloat, 32, 1 };
        m->dl_tensor.shape = new int64_t[2] { rows, cols };
        m->dl_tensor.strides = nullptr;
        m->dl_tensor.byte_offset = 0;
        m->manager_ctx = nullptr;
        m->deleter = counting_deleter;
        {
            FloatC x = FloatC::from_dlpack(m);
            CHECK(x.data() == dev && x.size() == (size_t) count);
            FloatC y = x * x + 1.f;
            std::vector<float> got = host(y);
            for (int64_t i = 0; i < count; ++i) CHECK(got[i] == xf[i] * xf[i] + 1.f);
            CHECK(g_deleted == 0);
        }
        cuda_sync();
        CHECK(g_deleted == 1);
        cuda_sync();
        CHECK(g_deleted == 1);
    }
    printf("dlpack_check ok\n");
    return 0;
}
