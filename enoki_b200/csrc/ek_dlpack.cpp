/*
 * ek_dlpack.cpp -- zero-copy exchange of device buffers through DLPack (no counterpart in the reference, which copies
 * in both directions: src/python/common.h:1085-1215).
 *
 * The runtime has no locks and belongs to one thread, but a consumer drops an exported tensor on whichever thread
 * releases its last reference (torch: autograd workers, the garbage collector).  So the export's deleter touches no
 * runtime state: it records an event on the consumer's stream and queues (handle, event) under a mutex of its own.
 * The owning thread drains that queue at its next entry into the runtime, makes the backend's stream wait on the event
 * and drops the reference.  Imports go the other way: a freed import records an event on the backend's stream and the
 * producer's deleter is called once that event has completed, on the owning thread.
 */
#include "ek_internal.h"
#include "../../include/enoki_b200_dlpack.h"
#include <mutex>
#include <string>
#include <vector>

std::atomic<uint32_t> ek_dlpack_pending { 0 };

namespace {

struct Released { uint32_t handle; uint64_t epoch; cudaEvent_t event; };
struct FreedImport { void *managed; bool versioned; cudaEvent_t event; };

std::mutex g_mutex;
std::vector<Released> g_released;        /* guarded by g_mutex: exports dropped by their consumer */
std::vector<FreedImport> g_freed;        /* owning thread only: imports whose producer is told once `event` completed */
std::atomic<uint64_t> g_epoch { 0 };     /* bumped by ek_shutdown: handles of earlier contexts are void */

/* what an export's manager_ctx points to */
struct ExportCtx {
    int64_t shape[1];
    uint32_t handle;
    int device;
    uint64_t epoch;
    cudaStream_t consumer;
};

bool dtype_of(ek_type t, DLDataType &d) {
    d.lanes = 1;
    d.bits = (uint8_t) (8 * ek_type_size(t));
    switch (t) {
        case EK_INT8: case EK_INT16: case EK_INT32: case EK_INT64: d.code = kDLInt; return true;
        case EK_UINT8: case EK_UINT16: case EK_UINT32: case EK_UINT64: d.code = kDLUInt; return true;
        case EK_FLOAT16: case EK_FLOAT32: case EK_FLOAT64: d.code = kDLFloat; return true;
        case EK_BOOL: d.code = kDLBool; return true;
        default: return false;
    }
}

/* the exact inverse of dtype_of; EK_INVALID for anything else */
ek_type type_of(DLDataType d) {
    static const ek_type ints[] = { EK_INT8, EK_INT16, EK_INT32, EK_INT64 }, uints[] = { EK_UINT8, EK_UINT16, EK_UINT32, EK_UINT64 },
                         floats[] = { EK_INVALID, EK_FLOAT16, EK_FLOAT32, EK_FLOAT64 };
    int k = d.bits == 8 ? 0 : d.bits == 16 ? 1 : d.bits == 32 ? 2 : d.bits == 64 ? 3 : -1;
    if (k < 0) return EK_INVALID;
    switch (d.code) {
        case kDLInt: return ints[k];
        case kDLUInt: return uints[k];
        case kDLFloat: return floats[k];
        case kDLBool: return d.bits == 8 ? EK_BOOL : EK_INVALID;
        default: return EK_INVALID;
    }
}

std::string dtype_name(DLDataType d) {
    const char *names[] = { "int", "uint", "float", "opaque handle", "bfloat", "complex", "bool" };
    if (d.code <= kDLBool) return names[d.code] + std::to_string(d.bits);
    if (d.code <= 14) return "float8 (type code " + std::to_string(d.code) + ")";   /* DLPack 1.1's float8 formats */
    return "of type code " + std::to_string(d.code) + " and " + std::to_string(d.bits) + " bits";
}

template <typename M> void export_deleter(M *self) {
    /* any thread: no runtime call here */
    ExportCtx *c = (ExportCtx *) self->manager_ctx;
    cudaEvent_t ev = nullptr;
    if (c->consumer) {
        int prev = -1;
        cudaGetDevice(&prev);
        if (prev != c->device) cudaSetDevice(c->device);
        if (cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) != cudaSuccess || cudaEventRecord(ev, c->consumer) != cudaSuccess) {
            /* no event: wait for the consumer's work here instead */
            cudaGetLastError();
            if (ev) { cudaEventDestroy(ev); ev = nullptr; }
            cudaStreamSynchronize(c->consumer);
        }
        if (prev >= 0 && prev != c->device) cudaSetDevice(prev);
    }
    {
        std::lock_guard<std::mutex> lock(g_mutex);
        g_released.push_back({ c->handle, c->epoch, ev });
        ek_dlpack_pending.fetch_add(1, std::memory_order_release);
    }
    delete c;
    delete self;
}

template <typename M> M *make_export(uint32_t index, const EkVariable &v, const DLDataType &dt, cudaStream_t consumer) {
    M *m = new M();
    ExportCtx *c = new ExportCtx();
    c->shape[0] = (int64_t) v.size;
    c->handle = index;
    c->device = ek_planned_device();
    c->epoch = g_epoch.load();
    c->consumer = consumer;
    DLTensor &t = m->dl_tensor;
    t.data = v.data;
    t.device = { kDLCUDA, c->device };
    t.ndim = 1;
    t.dtype = dt;
    t.shape = c->shape;
    t.strides = nullptr;
    t.byte_offset = 0;
    m->manager_ctx = c;
    m->deleter = export_deleter<M>;
    return m;
}

void call_deleter(void *managed, bool versioned) {
    if (versioned) { auto *m = (DLManagedTensorVersioned *) managed; if (m->deleter) m->deleter(m); }
    else { auto *m = (DLManagedTensor *) managed; if (m->deleter) m->deleter(m); }
}

bool refuse(const std::string &why) {
    ek_set_error("ek_dlpack_import(): " + why);
    return false;
}

/* every check of an import, before any CUDA call */
bool check_import(const DLTensor &t, ek_type &type, size_t &size) {
    if (t.device.device_type != kDLCUDA)
        return refuse("device type " + std::to_string((int) t.device.device_type) +
                      " is not supported: only CUDA device memory (kDLCUDA) can be aliased");
    int dev = ek_planned_device();
    if (t.device.device_id != dev)
        return refuse("the tensor is on CUDA device " + std::to_string(t.device.device_id) + ", the backend runs on device " +
                      std::to_string(dev));
    if (t.dtype.lanes != 1)
        return refuse("dtype with " + std::to_string(t.dtype.lanes) + " lanes is not supported (lanes must be 1)");
    type = type_of(t.dtype);
    if (type == EK_INVALID) return refuse("dtype " + dtype_name(t.dtype) + " is not supported");
    if (t.ndim < 0 || (t.ndim > 0 && !t.shape)) return refuse("invalid shape (ndim " + std::to_string(t.ndim) + ")");
    uint64_t n = 1;
    for (int i = 0; i < t.ndim; ++i) {
        if (t.shape[i] < 0) return refuse("invalid shape (extent " + std::to_string(t.shape[i]) + ")");
        if (t.shape[i] == 0) return refuse("size zero: empty tensors cannot be imported");
        if ((uint64_t) t.shape[i] > 0xffffffffull || n * (uint64_t) t.shape[i] > 0xffffffffull)
            return refuse("size: arrays with more than 2^32-1 entries are not supported");
        n *= (uint64_t) t.shape[i];
    }
    if (t.strides) {
        int64_t expect = 1;
        for (int i = t.ndim - 1; i >= 0; --i) {
            if (t.shape[i] != 1 && t.strides[i] != expect)
                return refuse("strides are not C-contiguous (dimension " + std::to_string(i) + " has stride " +
                              std::to_string(t.strides[i]) + ", a compact row-major layout needs " + std::to_string(expect) +
                              "): call .contiguous() first");
            expect *= t.shape[i];
        }
    }
    if (!t.data) return refuse("null data pointer");
    size_t es = ek_type_size(type);
    if (((uintptr_t) t.data + t.byte_offset) % es != 0)
        return refuse("data is not aligned to its " + std::to_string(es) + "-byte elements");
    size = (size_t) n;
    return true;
}

} // namespace

void ek_dlpack_release_import(EkVariable &v) {
    EkContext &ctx = ek_ctx();
    cudaEvent_t ev = nullptr;
    if (ctx.initialized) {      /* (before ek_init no work can have been enqueued on the buffer) */
        ek_cuda_check(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        ek_cuda_check(cudaEventRecord(ev, ctx.stream));
    }
    g_freed.push_back({ v.dlpack, v.dlpack_versioned, ev });
    ek_dlpack_pending.fetch_add(1, std::memory_order_release);
    v.dlpack = nullptr;
    v.data = nullptr;
}

void ek_dlpack_drain_slow(bool wait) {
    std::vector<Released> released;
    {
        std::lock_guard<std::mutex> lock(g_mutex);
        released.swap(g_released);
        ek_dlpack_pending.fetch_sub((uint32_t) released.size(), std::memory_order_relaxed);
    }
    EkContext &ctx = ek_ctx();
    for (const Released &r : released) {
        if (r.event) {
            if (ctx.initialized) ek_cuda_check(cudaStreamWaitEvent(ctx.stream, r.event, 0));
            cudaEventDestroy(r.event);
        }
        if (r.epoch == g_epoch.load()) ek_dec_ref_ext(r.handle);   /* may free imports: they join g_freed */
    }
    /* the producers' deleters run last: they may re-enter (a torch tensor exported by this backend queues its release) */
    std::vector<FreedImport> done;
    size_t keep = 0;
    for (const FreedImport &f : g_freed) {
        bool ready = true;
        if (f.event) {
            cudaError_t err = wait ? cudaEventSynchronize(f.event) : cudaEventQuery(f.event);
            if (err == cudaErrorNotReady) { cudaGetLastError(); ready = false; }
            else { ek_cuda_check(err); cudaEventDestroy(f.event); }
        }
        if (ready) done.push_back(f); else g_freed[keep++] = f;
    }
    g_freed.resize(keep);
    ek_dlpack_pending.fetch_sub((uint32_t) done.size(), std::memory_order_relaxed);
    for (const FreedImport &f : done) call_deleter(f.managed, f.versioned);
    /* a deleter may have queued another release (an import of this backend's own export): drain that too */
    if (wait && ek_dlpack_pending.load(std::memory_order_acquire)) ek_dlpack_drain_slow(true);
}

void ek_dlpack_shutdown() {
    ek_dlpack_drain(true);
    g_epoch.fetch_add(1);
}

extern "C" {

int ek_device(void) { return ek_planned_device(); }

void *ek_dlpack_export(uint32_t index, int versioned, void *consumer_stream) {
    ek_dlpack_drain();
    EkContext &ctx = ek_ctx();
    if (index < EK_REG_RESERVED || index >= ctx.vars.size() || !ctx.vars[index].used) {
        ek_set_error("ek_dlpack_export(): unknown variable " + std::to_string(index));
        return nullptr;
    }
    DLDataType dt;
    if (!dtype_of(ctx.vars[index].type, dt)) {
        ek_set_error(std::string("ek_dlpack_export(): arrays of type ") + ek_type_name(ctx.vars[index].type) +
                     " cannot be exported (DLPack has no pointer type)");
        return nullptr;
    }
    if (ek_eval_var(index) != 0) return nullptr;
    const EkVariable &v = ctx.vars[index];
    if (!v.data) { ek_set_error("ek_dlpack_export(): variable has no storage"); return nullptr; }
    ek_inc_ref_ext(index);
    if (versioned) {
        DLManagedTensorVersioned *m = make_export<DLManagedTensorVersioned>(index, v, dt, (cudaStream_t) consumer_stream);
        m->version = { DLPACK_MAJOR_VERSION, DLPACK_MINOR_VERSION };
        m->flags = 0;
        return m;
    }
    return make_export<DLManagedTensor>(index, v, dt, (cudaStream_t) consumer_stream);
}

uint32_t ek_dlpack_import(void *managed, int versioned) {
    ek_dlpack_drain();
    if (!managed) { ek_set_error("ek_dlpack_import(): null tensor"); return 0; }
    const DLTensor *t;
    if (versioned) {
        const DLManagedTensorVersioned *m = (const DLManagedTensorVersioned *) managed;
        if (m->version.major != DLPACK_MAJOR_VERSION) {
            ek_set_error("ek_dlpack_import(): DLPack version " + std::to_string(m->version.major) + "." +
                         std::to_string(m->version.minor) + " is not supported (major version 1 is)");
            return 0;
        }
        if (m->flags & DLPACK_FLAG_BITMASK_READ_ONLY) {
            ek_set_error("ek_dlpack_import(): read-only tensors are not supported (arrays are writable)");
            return 0;
        }
        t = &m->dl_tensor;
    } else {
        t = &((const DLManagedTensor *) managed)->dl_tensor;
    }
    ek_type type = EK_INVALID; size_t size = 0;
    if (!check_import(*t, type, size)) return 0;
    uint32_t idx = ek_var_register(type, size, (uint8_t *) t->data + t->byte_offset, 0);
    if (!idx) return 0;
    EkVariable &v = ek_ctx().vars[idx];
    v.dlpack = managed;
    v.dlpack_versioned = versioned != 0;
    return idx;
}

int ek_stream_wait_external(void *stream) {
    EkContext &ctx = ek_ctx();
    if (ek_init() != 0) return -1;
    if (!ctx.handoff_event) ek_cuda_check(cudaEventCreateWithFlags(&ctx.handoff_event, cudaEventDisableTiming));
    ek_cuda_check(cudaEventRecord(ctx.handoff_event, (cudaStream_t) stream));
    ek_cuda_check(cudaStreamWaitEvent(ctx.stream, ctx.handoff_event, 0));
    return 0;
}

int ek_stream_signal_external(void *stream) {
    EkContext &ctx = ek_ctx();
    if (ek_init() != 0) return -1;
    if (!ctx.handoff_event) ek_cuda_check(cudaEventCreateWithFlags(&ctx.handoff_event, cudaEventDisableTiming));
    ek_cuda_check(cudaEventRecord(ctx.handoff_event, ctx.stream));
    ek_cuda_check(cudaStreamWaitEvent((cudaStream_t) stream, ctx.handoff_event, 0));
    return 0;
}

} /* extern "C" */
