/*
 * enoki_b200_dlpack.h -- the DLPack exchange structures (ABI version 1.0), written from the public DLPack
 * specification.  Only what ek_dlpack_export() / ek_dlpack_import() exchange is declared.
 *
 * The include guard is dlpack.h's own: whichever of the two headers a translation unit includes first declares the
 * structures (they are the same ABI), and the other is skipped.  libtorch's ATen/dlpack.h is such a header.
 */
#ifndef DLPACK_DLPACK_H_
#define DLPACK_DLPACK_H_

#include <stdint.h>

#define DLPACK_MAJOR_VERSION 1
#define DLPACK_MINOR_VERSION 0

/* DLManagedTensorVersioned::flags */
#define DLPACK_FLAG_BITMASK_READ_ONLY (1ULL << 0)
#define DLPACK_FLAG_BITMASK_IS_COPIED (1ULL << 1)

#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
    uint32_t major;
    uint32_t minor;
} DLPackVersion;

typedef enum {
    kDLCPU = 1,
    kDLCUDA = 2,
    kDLCUDAHost = 3,
    kDLOpenCL = 4,
    kDLVulkan = 7,
    kDLMetal = 8,
    kDLVPI = 9,
    kDLROCM = 10,
    kDLROCMHost = 11,
    kDLExtDev = 12,
    kDLCUDAManaged = 13,
    kDLOneAPI = 14,
    kDLWebGPU = 15,
    kDLHexagon = 16
} DLDeviceType;

typedef struct {
    DLDeviceType device_type;
    int32_t device_id;
} DLDevice;

typedef enum {
    kDLInt = 0,
    kDLUInt = 1,
    kDLFloat = 2,
    kDLOpaqueHandle = 3,
    kDLBfloat = 4,
    kDLComplex = 5,
    kDLBool = 6
} DLDataTypeCode;

typedef struct {
    uint8_t code;       /* a DLDataTypeCode */
    uint8_t bits;
    uint16_t lanes;
} DLDataType;

typedef struct {
    void *data;
    DLDevice device;
    int32_t ndim;
    DLDataType dtype;
    int64_t *shape;
    int64_t *strides;   /* in elements; NULL = compact row-major */
    uint64_t byte_offset;
} DLTensor;

typedef struct DLManagedTensor {
    DLTensor dl_tensor;
    void *manager_ctx;
    void (*deleter)(struct DLManagedTensor *self);
} DLManagedTensor;

typedef struct DLManagedTensorVersioned {
    DLPackVersion version;
    void *manager_ctx;
    void (*deleter)(struct DLManagedTensorVersioned *self);
    uint64_t flags;
    DLTensor dl_tensor;
} DLManagedTensorVersioned;

#ifdef __cplusplus
}
#endif
#endif /* DLPACK_DLPACK_H_ */
