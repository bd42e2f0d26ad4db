"""Where the oracle's native libraries live, when they are built and how they are opened (TEST INFRASTRUCTURE ONLY).

  oracle/liborb_oracle.so   every C restatement; brought up to date by oracle/Makefile (oracle.build()) before it is opened
  oracle/_ref/lib*.so       the drivers of the reference's own code, opened RTLD_NOW | RTLD_LOCAL as they are; only a
                            missing one is built, by `make ref` (oracle.ref.build(), where the reference sources exist)

Opening the C oracle never builds the reference."""
import ctypes as C
import functools
import os

HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(HERE, "_ref")


def p(a):
    """The address of numpy array `a` as a void* argument; None for NULL."""
    return None if a is None else a.ctypes.data_as(C.c_void_p)


@functools.cache
def _open(name):
    path = os.path.join(HERE, name)
    if not name.startswith("_ref/"):
        from . import build
        build()
        return C.CDLL(path)
    if not os.path.exists(path):
        from . import ref
        ref.build()
    return C.CDLL(path, mode=os.RTLD_NOW | os.RTLD_LOCAL)


def loader(name, sigs, optional=()):
    """A function returning oracle/<name> ("liborb_oracle.so" or "_ref/lib*.so") with the signature table
    {function: (restype, [argtypes])} applied.  A library is opened once per name; each table is applied on its first call.
    The functions named in `optional` may be absent (a prebuilt _ref/ library older than its driver source, where the
    reference sources to rebuild it are not present): they are left unbound, so `has(lib, f)` is False; every other
    function of the table must be there."""
    @functools.cache
    def lib():
        L = _open(name)
        for f, (restype, argtypes) in sigs.items():
            if f in optional and not hasattr(L, f):
                continue
            fn = getattr(L, f)
            fn.restype, fn.argtypes = restype, argtypes
        return L
    return lib


def has(lib, f):
    """whether the library returned by loader function `lib` exports function `f`"""
    return hasattr(lib(), f)


def ref_available(name):
    """oracle/_ref/<name> and the reference library it links against are both built."""
    return os.path.exists(os.path.join(REF_DIR, name)) and os.path.exists(os.path.join(REF_DIR, "libref_orbslam.so"))
