"""CPU: the entry points of prompts padded to a capacity (ape_gemm_tn_cols_dev, ape_vlf_fold_vision_dev, ape_vlf_fold_pool_dev)
check their arguments before any launch, so no device is needed."""
import ctypes
import threading


def test_bad_arguments_are_reported(built):
    """The calls run on a thread of their own: the error text is thread-local, so this thread's stays as it was."""
    from ape_b200 import _lib

    lib = _lib.lib
    n_dev = ctypes.c_int(3)  # host memory: never read, every call below fails first
    buf = ctypes.create_string_buffer(64)
    a = ctypes.addressof(buf) + (-ctypes.addressof(buf)) % 16  # 16-byte aligned, never read
    cases = [
        ((a, 256, a, 256, a, 64, None, 20, 64, 256, ctypes.addressof(n_dev), 7, None), -1, b"dtype 7"),
        ((a, 256, a, 256, a, 64, None, 20, 0, 256, ctypes.addressof(n_dev), 1, None), -1, b"N=0"),
        ((a, 256, a, 256, a, 64, None, -1, 64, 256, ctypes.addressof(n_dev), 1, None), -1, b"M=-1"),
        ((a, 256, a, 256, a, 64, None, 20, 64, 256, None, 1, None), -3, b"null pointer"),
        ((a + 2, 256, a, 256, a, 64, None, 20, 64, 256, ctypes.addressof(n_dev), 1, None), -1, b"16-byte"),
        ((a, 256, a, 256, a, 32, None, 20, 64, 256, ctypes.addressof(n_dev), 2, None), -1, b"row pitch"),
        ((a, 256, a, 256, a, 64, None, 20, 64, 256, ctypes.addressof(n_dev) + 1, 2, None), -1, b"4-byte"),
    ]
    seen = []

    def run():
        for args, _, _ in cases:
            rc = lib.ape_gemm_tn_cols_dev(*args)
            seen.append((rc, lib.ape_last_error()))

    t = threading.Thread(target=run)
    t.start()
    t.join()
    for (rc, msg), (_, want_rc, want_msg) in zip(seen, cases):
        assert rc == want_rc and want_msg in msg, (rc, msg)


def test_fold_dev_bad_arguments_are_reported(built):
    """ape_vlf_fold_vision_dev / ape_vlf_fold_pool_dev check the device count pointer and the shapes before any launch."""
    from ape_b200 import _lib

    lib = _lib.lib
    n_dev = ctypes.c_int(3)
    buf = ctypes.create_string_buffer(64)
    a = ctypes.addressof(buf) + (-ctypes.addressof(buf)) % 16
    nd = ctypes.addressof(n_dev)
    vision = lambda n_ptr, N, dtype: lib.ape_vlf_fold_vision_dev(a, 256, a, a, a, a, a, a, 256, 1, 64, N, 8, n_ptr, 256, dtype,  # noqa: E731
                                                                 None)
    pool = lambda n_ptr, N, dtype: lib.ape_vlf_fold_pool_dev(a, 256, a, a, a, 2048, 1, 64, N, 8, n_ptr, 256, dtype, None)  # noqa: E731
    cases = [(vision, (None, 16, 1), -3, b"null n_dev"), (vision, (nd + 1, 16, 1), -1, b"4-byte"), (vision, (nd, 16, 7), -1, b"fp16"),
             (vision, (nd, 0, 1), -2, b"N=0"), (pool, (None, 16, 1), -3, b"null n_dev"), (pool, (nd + 2, 16, 2), -1, b"4-byte"),
             (pool, (nd, 16, 0), -1, b"fp16"), (pool, (nd, 0, 2), -2, b"N=0")]
    seen = []

    def run():
        for fn, args, _, _ in cases:
            seen.append((fn(*args), lib.ape_last_error()))

    t = threading.Thread(target=run)
    t.start()
    t.join()
    for (rc, msg), (_, _, want_rc, want_msg) in zip(seen, cases):
        assert rc == want_rc and want_msg in msg, (rc, msg)
