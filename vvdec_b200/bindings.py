"""ctypes prototypes for libvvdec_b200.so (include/vvdec_b200.h)."""
import ctypes as C
import numpy as np
from . import abi

i16p = np.ctypeslib.ndpointer(np.int16, flags="C_CONTIGUOUS")
PLANES = C.POINTER(C.POINTER(C.c_int16))


def declare(lib):
    lib.b200_last_error.restype = C.c_char_p
    lib.b200_version.restype = C.c_char_p
    lib.b200_device_count.restype = C.c_int
    lib.b200_k1_residual.argtypes = [C.POINTER(abi.Geom), PLANES, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                     C.c_void_p, C.c_size_t, C.c_int]
    lib.b200_k1_residual.restype = C.c_int


    lib.b200_lf_deblock.argtypes = [C.POINTER(abi.Geom), PLANES, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                    C.c_void_p, C.c_int]
    lib.b200_lf_deblock.restype = C.c_int
    lib.b200_lf_derive.argtypes = [C.POINTER(abi.Geom), C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t,
                                   C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    lib.b200_lf_derive.restype = C.c_int


    lib.b200_sao_picture.argtypes = [C.POINTER(abi.Geom), PLANES, PLANES, C.c_void_p, C.c_void_p]
    lib.b200_sao_picture.restype = C.c_int
    lib.b200_alf_picture.argtypes = [C.POINTER(abi.Geom), PLANES, PLANES, C.c_void_p, C.POINTER(abi.AlfTables)]
    lib.b200_alf_picture.restype = C.c_int


    lib.b200_mc_predict.argtypes = [C.POINTER(abi.Geom), PLANES, C.POINTER(C.c_void_p), C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    lib.b200_mc_predict.restype = C.c_int
    lib.b200_mc_predict_wp.argtypes = [C.POINTER(abi.Geom), PLANES, C.POINTER(C.c_void_p), C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_int]
    lib.b200_mc_predict_wp.restype = C.c_int


    CTX = C.c_void_p
    lib.b200_ctx_create.argtypes = [C.POINTER(CTX), C.POINTER(abi.Geom), C.c_int, C.c_int, C.c_int]
    lib.b200_ctx_destroy.argtypes = [CTX]; lib.b200_ctx_destroy.restype = None
    lib.b200_ctx_load_slot.argtypes = [CTX, C.c_int, PLANES]
    lib.b200_decompress_picture.argtypes = [CTX, C.POINTER(abi.Picture)]
    lib.b200_pic_upload.argtypes = [CTX, C.POINTER(abi.Picture)]
    lib.b200_pic_run.argtypes = [CTX, C.c_int]
    lib.b200_wait_picture.argtypes = [CTX, C.c_int, C.c_void_p, C.c_size_t]
    lib.b200_get_frame.argtypes = [CTX, C.c_int, PLANES]
    lib.b200_get_frame_async.argtypes = [CTX, C.c_int, PLANES]
    lib.b200_ctx_load_slot_strided.argtypes = [CTX, C.c_int, PLANES, C.POINTER(C.c_ssize_t)]
    lib.b200_get_frame_strided.argtypes = [CTX, C.c_int, PLANES, C.POINTER(C.c_ssize_t)]
    lib.b200_frame_wait.argtypes = [CTX, C.c_int]
    lib.b200_get_frame_device_async.argtypes = [CTX, C.c_int, C.POINTER(C.c_void_p), C.c_void_p]
    lib.b200_frame_bytes.argtypes = [C.POINTER(abi.Geom), C.c_int, C.c_int]; lib.b200_frame_bytes.restype = C.c_size_t
    lib.b200_get_frame_fmt_async.argtypes = [CTX, C.c_int, C.c_int, C.POINTER(C.c_void_p)]
    lib.b200_intra_predict.argtypes = [C.POINTER(abi.Geom), PLANES, C.c_void_p, C.c_size_t]
    lib.b200_intra_reconstruct.argtypes = [C.POINTER(abi.Geom), PLANES, PLANES, C.c_void_p, C.c_size_t]
    lib.b200_frame_hash_async.argtypes = [CTX, C.c_int, C.c_int, C.c_void_p]
    lib.b200_get_frame_grain_async.argtypes = [CTX, C.c_int, C.c_int, C.POINTER(C.c_void_p), C.POINTER(abi.FilmGrain)]
    lib.b200_ctx_mark.argtypes = [CTX, C.c_int]
    lib.b200_ctx_elapsed_ms.argtypes = [CTX, C.POINTER(C.c_float)]
    lib.b200_ctx_kernel_launches.argtypes = [CTX]; lib.b200_ctx_kernel_launches.restype = C.c_longlong
    lib.b200_ctx_set_profiling.argtypes = [CTX, C.c_int]
    lib.b200_ctx_get_kernel_ms.argtypes = [CTX, C.POINTER(C.c_float), C.POINTER(C.c_int)]
    lib.b200_ctx_get_kernel_ms_n.argtypes = [CTX, C.POINTER(C.c_float), C.POINTER(C.c_int), C.c_int]
    lib.b200_host_register.argtypes = [C.c_void_p, C.c_size_t]
    lib.b200_host_unregister.argtypes = [C.c_void_p]


EXPORTS = ["b200_ctx_create", "b200_ctx_destroy", "b200_ctx_load_slot", "b200_decompress_picture", "b200_pic_upload", "b200_pic_run",
           "b200_wait_picture", "b200_get_frame", "b200_ctx_load_slot_strided", "b200_get_frame_strided", "b200_get_frame_async", "b200_get_frame_device_async", "b200_frame_wait", "b200_frame_bytes", "b200_get_frame_fmt_async", "b200_frame_hash_async", "b200_intra_predict", "b200_intra_reconstruct", "b200_get_frame_grain_async", "b200_ctx_mark", "b200_ctx_elapsed_ms", "b200_ctx_kernel_launches", "b200_ctx_set_profiling", "b200_ctx_get_kernel_ms", "b200_ctx_get_kernel_ms_n", "b200_host_register", "b200_host_unregister",
           "b200_mc_predict", "b200_mc_predict_wp", "b200_last_error", "b200_version", "b200_device_count", "b200_k1_residual", "b200_lf_deblock", "b200_lf_derive",
           "b200_sao_picture", "b200_alf_picture"]
