"""
setk_b200.libs.exraw -- the reference's dependency-free archive format for 1-D / 2-D ndarrays
(scripts/sptk/libs/exraw.py): per entry, "<key> " then a dtype flag (f / d / i / q), a shape flag
(v: one int32 length; m: two int32 dimensions) and the raw native-order bytes.  The same writer and
readers, with np.frombuffer where the reference calls the removed np.fromstring.
"""
import struct

import numpy as np

_FLAGS = {"float32": "f", "float64": "d", "int32": "i", "int64": "q"}
_DTYPES = {"f": (np.float32, 4), "d": (np.float64, 8), "i": (np.int32, 4), "q": (np.int64, 8)}


def _serialize(fd, arr):
    """exraw.py:13-34"""
    dtype = str(arr.dtype)
    if dtype not in _FLAGS:
        raise TypeError("Unsupported dtype: {}".format(arr.dtype))
    if arr.ndim >= 3:
        raise RuntimeError("Accept only 1/2D ndarray, got {:d}".format(arr.ndim))
    fd.write(str.encode(_FLAGS[dtype]))
    if arr.ndim == 1:
        fd.write(str.encode("v"))
        fd.write(struct.pack("i", arr.size))
    else:
        fd.write(str.encode("m"))
        M, N = arr.shape
        fd.write(struct.pack("i", M))
        fd.write(struct.pack("i", N))
    fd.write(arr.tobytes())


def _deserialize(fd, addr=None):
    """exraw.py:37-67"""
    if addr:
        fd.seek(addr)
    dtype = bytes.decode(fd.read(1))
    if dtype not in _DTYPES:
        raise TypeError("Unsupported dtype string, expect f/d/i/q, got {}".format(dtype))
    atype = bytes.decode(fd.read(1))
    if atype not in ["v", "m"]:
        raise TypeError("Unsupported atype string: expect v/m, got {}".format(atype))
    np_dtype, sizeof = _DTYPES[dtype]
    M, N = 0, 0
    if atype == "v":
        D = struct.unpack("i", fd.read(4))[0]
        raw = fd.read(D * sizeof)
    else:
        M, N = struct.unpack("ii", fd.read(8))
        raw = fd.read(M * N * sizeof)
    arr = np.frombuffer(raw, dtype=np_dtype).copy()
    return arr if atype == "v" else arr.reshape(M, N)


def _parse_scripts(scp):
    """exraw.py:70-92"""
    index_addr = dict()
    line = 0
    with open(scp, "r") as f:
        for raw_line in f:
            toks = raw_line.strip().split()
            line += 1
            if len(toks) != 2:
                raise RuntimeError("Content format error in {}:{:d}, {}".format(scp, line, raw_line))
            key, value = toks
            index_toks = value.split(":")
            if len(index_toks) != 2:
                raise RuntimeError("Value format error in {}:{:d}: {}".format(scp, line, raw_line))
            obj, shift = index_toks
            if key in index_addr:
                raise ValueError("Duplicated key '{}' exists in {}".format(key, index_addr))
            index_addr[key] = (obj, int(shift))
    return index_addr


class BinaryWriter(object):
    """exraw.py:95-132: writes `key ` + the serialised array; with scp, `key\\tobj:offset` lines."""

    def __init__(self, obj, scp=None):
        self.obj_str, self.scp_str = obj, scp
        if not self.obj_str:
            raise RuntimeError("BinaryWriter: Seems got empty object")

    def __enter__(self):
        self.obj = open(self.obj_str, "wb")
        self.scp = None if not self.scp_str else open(self.scp_str, "w")
        return self

    def __exit__(self, *args):
        self.obj.close()
        if self.scp:
            self.scp.close()

    def write(self, key, ndarray):
        if not isinstance(ndarray, np.ndarray):
            raise TypeError("Expect 2nd args as numpy's ndarray, but got type {}".format(type(ndarray)))
        if not isinstance(key, str):
            raise TypeError("Expect 1st args as python str object, but got type {}".format(type(key)))
        self.obj.write(str.encode(key + " "))
        offset = self.obj.tell()
        _serialize(self.obj, ndarray)
        if self.scp:
            self.scp.write("{0}\t{1}:{2}\n".format(key, self.obj_str, offset))


class BinaryObjectReader(object):
    """exraw.py:135-160: sequential (key, array) pairs of an archive."""

    def __init__(self, obj):
        self.obj_str = obj

    def _next_key(self, fd):
        key = ""
        while True:
            c = bytes.decode(fd.read(1))
            if c == " " or c == "":
                break
            key += c
        return key

    def __iter__(self):
        with open(self.obj_str, "rb") as fd:
            while True:
                key = self._next_key(fd)
                if not key:
                    break
                yield key, _deserialize(fd)


class BinaryScriptReader(object):
    """exraw.py:163-196: random access through an scp of `key obj:offset` lines."""

    def __init__(self, scp):
        self.index_addr = _parse_scripts(scp)
        self.mgr = dict()

    def __len__(self):
        return len(self.index_addr)

    def __contains__(self, key):
        return key in self.index_addr

    def __getitem__(self, key):
        return self._load(key)

    def __iter__(self):
        for key in self.index_addr:
            yield key, self._load(key)

    def _open(self, obj):
        if obj not in self.mgr:
            self.mgr[obj] = open(obj, "rb")
        return self.mgr[obj]

    def _load(self, key):
        obj, addr = self.index_addr[key]
        return _deserialize(self._open(obj), addr)

    def keys(self):
        return self.index_addr.keys()
