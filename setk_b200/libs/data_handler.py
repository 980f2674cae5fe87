"""
setk_b200.libs.data_handler -- Kaldi-style table readers / writers used by the
adaptive-beamformer CLI.  Public names and behaviour follow the reference's
scripts/sptk/libs/data_handler.py (parse_scps 139-170, Reader 173-236,
ScpReader 239-253, WaveReader 326-413, NumpyReader 439-448, SpectrogramReader
483-503, ScriptReader 506-535, WaveWriter 590-605, NumpyWriter 608-622); the
implementation is this repository's own.

Host-side IO is not the accelerated part (SURVEY.md section 8a "boundary
only").  What changes is SpectrogramReader: all channels of an utterance go
through ONE setk_stft launch instead of one librosa call per channel.
Kaldi archives: float / double matrices and vectors (tokens FM, DM, FV, DV) and the
compressed matrices CM / CM2 / CM3 (bit-identical to kaldi_io.py:248-318).
"""
import glob
import io
import os
import random
import struct
import subprocess
import sys
import warnings
from pathlib import Path

import numpy as np

from .utils import get_plan, read_wav, write_wav

__all__ = [
    "WaveWriter", "NumpyWriter", "SpectrogramReader", "ScriptReader", "WaveReader",
    "NumpyReader", "ScpReader", "Reader", "parse_scps"
]


# ------------------------------------------------------------------ streams ---
def _is_pipe(spec):
    return spec.rstrip().endswith("|")


def _shell_output(cmd):
    """stdout of a shell pipeline; raises with its stderr on failure."""
    done = subprocess.run(cmd, shell=True, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    if done.returncode != 0:
        raise Exception("There was an error while running the command "
                        f"\"{cmd}\":\n{done.stderr.decode(errors='replace')}\n")
    return done.stdout


class _Source(object):
    """Context manager over a path, "-" (stdin) or "command |" (pipe output)."""

    def __init__(self, spec, binary=False):
        self.spec = spec.strip()
        self.binary = binary
        self._owned = None

    def __enter__(self):
        if self.spec == "-":
            return sys.stdin.buffer if self.binary else sys.stdin
        if _is_pipe(self.spec):
            raw = _shell_output(self.spec[:-1])
            return io.BytesIO(raw) if self.binary else io.StringIO(raw.decode("utf-8"))
        if not os.path.exists(self.spec):
            raise FileNotFoundError(f"Could not find common file: \"{self.spec}\"")
        self._owned = open(self.spec, "rb") if self.binary else open(self.spec, "r",
                                                                      encoding="utf-8")
        return self._owned

    def __exit__(self, *exc):
        if self._owned is not None:
            self._owned.close()


def parse_scps(scp_path, value_processor=lambda x: x, num_tokens=2, restrict=True):
    """
    Kaldi script file -> {key: value}.  A line is `key value`, `key tok1 tok2 ...`
    (num_tokens != 2) or `key command ... |`; duplicate keys are an error.
    """
    table = {}
    with _Source(scp_path) as stream:
        for lineno, raw in enumerate(stream, 1):
            fields = raw.split()
            if not fields:
                continue
            key = fields[0]
            if fields[-1] == "|":
                value = " ".join(fields[1:])
            else:
                bad_count = num_tokens >= 2 and len(fields) != num_tokens
                if bad_count or (restrict and len(fields) < 2):
                    raise RuntimeError(f"For {scp_path}, format error in line[{lineno:d}]: {raw}")
                value = fields[1] if num_tokens == 2 else fields[1:]
            if key in table:
                raise ValueError(f"Duplicated key \'{key}\' exists in {scp_path}")
            table[key] = value_processor(value)
    return table


# ------------------------------------------------------------------ readers ---
class Reader(object):
    """Keyed, ordered collection with lazy loading: iteration yields (key, object)."""

    def __init__(self, index_dict):
        self.index_dict = index_dict
        self.index_keys = list(index_dict)

    def _load(self, key):
        return self.index_dict[key]

    def __len__(self):
        return len(self.index_keys)

    def __contains__(self, key):
        return key in self.index_dict

    def __iter__(self):
        return ((key, self._load(key)) for key in self.index_keys)

    def __getitem__(self, index):
        if isinstance(index, bool) or not isinstance(index, (int, str)):
            raise IndexError(f"Unsupported index type: {type(index)}")
        if isinstance(index, int):
            if not 0 <= index < len(self.index_keys):
                raise KeyError(f"Interger index out of range, {index:d} vs {len(self.index_keys):d}")
            index = self.index_keys[index]
        if index not in self.index_dict:
            raise KeyError(f"Missing utterance {index}!")
        return self._load(index)

    def get(self, index, default=None):
        return self[index] if index in self else default

    def sample(self, num_items):
        picked = [(k, self._load(k)) for k in random.sample(self.index_keys, num_items)]
        return picked[0] if num_items == 1 else picked


class ScpReader(Reader):
    """Reader over a Kaldi .scp table."""

    def __init__(self, scp_rspecifier, value_processor=lambda x: x, num_tokens=2, restrict=True):
        super().__init__(parse_scps(scp_rspecifier, value_processor, num_tokens, restrict))


class WaveReader(ScpReader):
    """
    wav.scp reader.  A value is a wav path, a glob over per-channel files (stacked
    in sorted order), `archive:offset`, or `command |` producing a wav on stdout.
    read() returns float32 samples, N or C x N.
    """

    def __init__(self, wav_scp, sr=16000, normalize=True, raw_pcm16=False):
        super().__init__(wav_scp)
        self.sr = sr
        self.normalize = normalize
        self.raw_pcm16 = raw_pcm16        # PCM-16 files come back as int16 (batched device feed)
        self._archives = {}

    def _decode(self, source, beg=None, end=None):
        return read_wav(source, beg=beg or 0, end=end, normalize=self.normalize, sr=self.sr,
                        raw_pcm16=self.raw_pcm16)

    def read_internal(self, addr, beg=None, end=None):
        if isinstance(addr, str) and ":" in addr:
            parts = addr.split(":")
            if len(parts) != 2:
                raise RuntimeError(f"Value format error: {addr}")
            handle = self._archives.get(parts[0])
            if handle is None:
                handle = self._archives[parts[0]] = open(parts[0], "rb")
            handle.seek(int(parts[1]))
            return self._decode(handle, beg, end)
        return self._decode(addr, beg, end)

    def read(self, key, beg=None, end=None):
        spec = self.index_dict[key].rstrip()
        if _is_pipe(spec):
            return self._decode(io.BytesIO(_shell_output(spec[:-1])))
        matches = sorted(glob.glob(spec))        # sorted: the channel order matters
        if not matches:
            raise RuntimeError(f"Could not find file matches template \'{spec}\'")
        channels = [self.read_internal(path, beg=beg, end=end) for path in matches]
        return channels[0] if len(channels) == 1 else np.vstack(channels)

    _load = read

    def maxabs(self, key):
        return np.max(np.abs(self.read(key)))

    def nsamps(self, key):
        return self.read(key).shape[-1]

    def duration(self, key):
        return self.nsamps(key) / self.sr

    def power(self, key):
        first = np.atleast_2d(self.read(key))[0]
        return np.linalg.norm(first, 2)**2 / first.size


class NumpyReader(ScpReader):
    """key -> numpy.load(path)."""

    def _load(self, key):
        return np.load(self.index_dict[key])


class SpectrogramReader(WaveReader):
    """
    wav.scp -> STFT: complex64 F x T (mono) or N x F x T, transposed to ... x T x F
    with transpose=True; keyword arguments are forward_stft's.
    """

    _defaults = dict(frame_len=1024, frame_hop=256, round_power_of_two=True, center=False,
                     window="hann", transpose=True)

    def __init__(self, wav_scp, normalize=True, **kwargs):
        super().__init__(wav_scp, normalize=normalize)
        self.stft_kwargs = kwargs

    def stft(self, samps, as_tensor=False):
        import torch
        from .utils import default_device
        opt = dict(self._defaults, **self.stft_kwargs)
        apply_abs, apply_log, apply_pow = (opt.pop(f, False) for f in ("apply_abs", "apply_log", "apply_pow"))
        if apply_log and not apply_abs:
            warnings.warn("Ignore apply_abs=False because apply_log=True")
            apply_abs = True
        if apply_pow and not apply_abs:
            raise NotImplementedError("SpectrogramReader: apply_pow of the complex STFT is not supported here")
        x = np.ascontiguousarray(np.atleast_2d(samps), dtype=np.float32)
        dev = default_device()
        plan = get_plan(x.shape[0], opt["frame_len"], opt["frame_hop"], opt["center"],
                        opt["round_power_of_two"], opt["window"], x.shape[1], dev)
        x = torch.from_numpy(x).to(dev)[None]
        if apply_abs:       # forward_stft's abs / pow / log per channel (utils.py:130-135): N x T x F
            spec = plan.spectral_feats(x, apply_pow=apply_pow, apply_log=apply_log)[0]
            if not opt["transpose"]:
                spec = spec.transpose(-1, -2)
        else:
            spec = plan.stft(x)[0]                                         # N x F x T
            if opt["transpose"]:
                spec = spec.transpose(-1, -2)
        if samps.ndim == 1:
            spec = spec[0]
        return spec if as_tensor else spec.cpu().numpy()

    def _load(self, key):
        return self.stft(self.read(key))


def _read_compressed_matrix(fd, token):
    """
    Kaldi CompressedMatrix (kaldi_io.py:248-318): global header {min, range, rows, cols};
    CM  = per-column header of four uint16 percentiles + one uint8 per element (column major),
    CM2 = uint16 per element, CM3 = uint8 per element (row major).  Same float32 arithmetic
    as the reference's uncompress().
    """
    min_val, prange, num_rows, num_cols = struct.unpack("<ffii", fd.read(16))
    if token == "CM":
        raw = fd.read(num_cols * (8 + num_rows))
        if len(raw) != num_cols * (8 + num_rows):
            raise RuntimeError("truncated compressed Kaldi matrix")
        pch = np.frombuffer(raw[:8 * num_cols], dtype="<u2").astype(np.float32)
        pch = np.transpose(pch.reshape(num_cols, 4))
        pch = pch * prange / 65535.0 + min_val
        u8 = np.frombuffer(raw[8 * num_cols:], dtype=np.uint8).astype(np.float32)
        u8 = np.transpose(u8.reshape(num_cols, num_rows))
        return np.where(
            u8 <= 64, u8 * (pch[1] - pch[0]) / 64.0 + pch[0],
            np.where(u8 >= 193, (u8 - 192) * (pch[3] - pch[2]) / 63.0 + pch[2],
                     (u8 - 64) * (pch[2] - pch[1]) / 128.0 + pch[1]))
    if token == "CM2":
        seq = np.frombuffer(fd.read(2 * num_rows * num_cols), dtype="<u2").astype(np.float32)
        inc = float(prange / 65535.0)
    else:
        seq = np.frombuffer(fd.read(num_rows * num_cols), dtype=np.uint8).astype(np.float32)
        inc = float(prange / 255.0)
    return min_val + seq.reshape(num_rows, num_cols) * inc


def compress_kaldi_cm(mat):
    """
    float32 matrix [rows][cols] -> the bytes of a Kaldi CompressedMatrix of format "CM" as they
    follow the "CM " token in an archive (global header, per-column percentile headers, one byte
    per element, column major) -- what Kaldi's copy-feats --compress=true writes and what
    _read_compressed_matrix / setk_cm_masks expand.  The percentiles of a column are its minimum,
    quartiles and maximum (kept strictly increasing as 16-bit codes, like Kaldi does); an element
    becomes the nearest code of its segment.
    """
    mat = np.ascontiguousarray(mat, dtype=np.float32)
    rows, cols = mat.shape
    min_val = float(mat.min()) if mat.size else 0.0
    prange = float(mat.max()) - min_val if mat.size else 1.0
    if not prange > 0.0:
        prange = 1.0
    q = np.quantile(mat, [0.0, 0.25, 0.75, 1.0], axis=0) if rows else np.zeros((4, cols))
    code = np.clip(np.rint((q - min_val) / prange * 65535.0), 0, 65535).astype(np.int64)
    code[0] = np.minimum(code[0], 65532)
    for i in (1, 2, 3):
        code[i] = np.clip(np.maximum(code[i], code[i - 1] + 1), 0, 65532 + i)
    pch = code.astype(np.float32) * np.float32(prange) / np.float32(65535.0) + np.float32(min_val)
    p0, p1, p2, p3 = (pch[i][None, :] for i in range(4))
    with np.errstate(invalid="ignore", divide="ignore"):
        lo = np.clip(np.rint((mat - p0) / (p1 - p0) * 64.0), 0, 64)
        mid = np.clip(64 + np.rint((mat - p1) / (p2 - p1) * 128.0), 64, 192)
        hi = np.clip(192 + np.rint((mat - p2) / (p3 - p2) * 63.0), 192, 255)
    u8 = np.where(mat < p1, lo, np.where(mat < p2, mid, hi)).astype(np.uint8)
    return (struct.pack("<ffii", min_val, prange, rows, cols) + code.T.astype("<u2").tobytes() +
            np.ascontiguousarray(u8.T).tobytes())


def read_kaldi_matrix(fd):
    """
    One uncompressed Kaldi float/double matrix or vector from a binary stream
    positioned at the "\\0B" marker (where an scp's `archive:offset` points).
    """
    if fd.read(2) != b"\0B":
        raise RuntimeError("Kaldi object is not in binary mode")
    token = bytearray()
    while True:
        ch = fd.read(1)
        if ch in (b" ", b""):
            break
        token += ch
    token = token.decode()
    if token in ("CM", "CM2", "CM3"):
        return _read_compressed_matrix(fd, token)
    if token not in ("FM", "DM", "FV", "DV"):
        raise RuntimeError(f"Unknown Kaldi object token: {token}")
    dtype = np.dtype("<f4" if token[0] == "F" else "<f8")

    def int32():
        marker, value = struct.unpack("<bi", fd.read(5))
        if marker != 4:
            raise RuntimeError("Kaldi int32 size marker expected")
        return value

    shape = (int32(), int32()) if token[1] == "M" else (int32(),)
    count = int(np.prod(shape))
    return np.frombuffer(fd.read(count * dtype.itemsize), dtype=dtype).reshape(shape).copy()


class ScriptReader(ScpReader):
    """feats.scp-style reader: key -> matrix at `archive:offset`."""

    def __init__(self, ark_scp):

        def split_address(addr):
            path, sep, offset = addr.rpartition(":")
            if not sep:
                raise ValueError("Unsupported scripts address format")
            return path, int(offset)

        super().__init__(ark_scp, value_processor=split_address)
        self._archives = {}

    def _load(self, key):
        path, offset = self.index_dict[key]
        handle = self._archives.get(path)
        if handle is None:
            handle = self._archives[path] = open(path, "rb")
        handle.seek(offset)
        return read_kaldi_matrix(handle)


# ------------------------------------------------------------------ writers ---
class Writer(object):
    """Directory-of-files writer with an optional `key<TAB>path` script."""

    def __init__(self, obj_path_or_dir, scp_path=None, is_dir=False):
        self.scp_path = scp_path
        if obj_path_or_dir == "-" and scp_path:        # data_handler.py:278-281
            warnings.warn("Ignore script output discriptor cause dump archives to stdout")
            self.scp_path = None
        self.dump_out_dir = is_dir
        if is_dir:
            self.path_or_dir = Path(obj_path_or_dir).absolute()
            self.path_or_dir.mkdir(exist_ok=True, parents=True)
        else:
            self.path_or_dir = "-" if obj_path_or_dir == "-" else os.path.abspath(obj_path_or_dir)
        self.scp_file = None
        self.ark_file = None

    def __enter__(self):
        if not self.dump_out_dir:                       # "wb" is important
            self.ark_file = sys.stdout.buffer if self.path_or_dir == "-" else open(self.path_or_dir, "wb")
        if self.scp_path:
            self.scp_file = sys.stdout if self.scp_path == "-" else open(self.scp_path, "w",
                                                                         encoding="utf-8")
        return self

    def __exit__(self, *exc):
        if self.ark_file is not None and self.ark_file is not sys.stdout.buffer:
            self.ark_file.close()
        if self.scp_file is not None and self.scp_file is not sys.stdout:
            self.scp_file.close()

    def check_args(self, data):
        if not isinstance(data, np.ndarray):
            raise RuntimeError(f"Instance of Writer accepts np.ndarray object, but got {type(data)}")

    def _record(self, key, path):
        if self.scp_file is not None:
            self.scp_file.write(f"{key}\t{path}\n")

    def write(self, key, data):
        raise NotImplementedError


class WaveWriter(Writer):
    """<dump_dir>/<key>.wav, PCM-16 like soundfile's default."""

    def __init__(self, dump_dir, scp_path=None, sr=16000, normalize=True):
        super().__init__(dump_dir, scp_path, is_dir=True)
        self.sr = sr
        self.normalize = normalize

    def write(self, key, obj):
        self.check_args(obj)
        target = self.path_or_dir / f"{key}.wav"
        write_wav(target, obj, sr=self.sr, normalize=self.normalize)
        self._record(key, target)


class NumpyWriter(Writer):
    """<dump_dir>/<key>.npy"""

    def __init__(self, dump_dir, scp_path=None):
        super().__init__(dump_dir, scp_path, is_dir=True)

    def write(self, key, obj):
        self.check_args(obj)
        target = self.path_or_dir / f"{key}.npy"
        np.save(target, obj)
        self._record(key, target)


def write_kaldi_matrix(fd, mat):
    """
    Kaldi binary float matrix / vector (kaldi_io.py:156-168, 218-229, 351-361):
    token FM|DM (FV|DV), then \\4 + int32 sizes, then the raw row-major data.
    """
    if not isinstance(mat, np.ndarray):
        raise TypeError(f"Unsupport type: {type(mat)}")
    if mat.dtype not in (np.float32, np.float64):
        raise AssertionError("kaldi archives hold float32 / float64 data")
    double = mat.dtype == np.float64
    if mat.ndim == 2:
        fd.write(b"DM " if double else b"FM ")
        fd.write(b"\x04" + struct.pack("i", mat.shape[0]))
        fd.write(b"\x04" + struct.pack("i", mat.shape[1]))
    elif mat.ndim == 1:
        fd.write(b"DV " if double else b"FV ")
        fd.write(b"\x04" + struct.pack("i", mat.size))
    else:
        raise RuntimeError(f"Only support 2D matrix, but got {mat.ndim:d}")
    fd.write(np.ascontiguousarray(mat).tobytes())


class ArchiveWriter(Writer):
    """
    Writer for kaldi's scripts && archive (BaseFloat matrix): data_handler.py:564-587.
    Each entry is `key ` + `\\0B` + the binary matrix; the script line points at the
    offset of the binary marker (`key<TAB>path:offset`).
    """

    def __init__(self, ark_path, scp_path=None, dtype=np.float32):
        if not ark_path:
            raise RuntimeError("Seem configure path of archives as None")
        super().__init__(ark_path, scp_path)
        self.dtype = dtype

    def write(self, key, obj):
        self.check_args(obj)
        self.ark_file.write(str.encode(key + " "))
        offset = self.ark_file.tell() if self.path_or_dir != "-" else 0
        self.ark_file.write(b"\0B")
        write_kaldi_matrix(self.ark_file, obj.astype(self.dtype))
        if self.scp_file is not None:
            self.scp_file.write(f"{key}\t{self.path_or_dir}:{offset:d}\n")


# ------------------------------------------------- remaining table readers / writers ---
def read_kaldi_archive(fd):
    """(key, matrix | vector) for every entry of a binary Kaldi archive stream (kaldi_io.py:364-376)."""
    while True:
        token = bytearray()
        while True:
            ch = fd.read(1)
            if ch in (b" ", b""):
                break
            token += ch
        if not token:
            return
        yield token.decode().strip(), read_kaldi_matrix(fd)


class ArchiveReader(object):
    """Sequential reader of a Kaldi archive: a path, "-" (stdin) or "command |" (data_handler.py:311-323)."""

    def __init__(self, ark_or_pipe):
        self.ark_or_pipe = ark_or_pipe

    def __iter__(self):
        with _Source(self.ark_or_pipe, binary=True) as fd:
            yield from read_kaldi_archive(fd)


class DirReader(Reader):
    """Every `<obj_dir>/*.<prefix>` file, keyed by its file name (data_handler.py:256-267)."""

    def __init__(self, obj_dir, prefix):
        from .utils import filekey
        obj_dir = Path(obj_dir)
        if not obj_dir.is_dir():
            raise RuntimeError("DirReader expect directory as input")
        super().__init__({filekey(f): f for f in glob.glob((obj_dir / f"*.{prefix}").as_posix())})


class SegmentWaveReader(ScpReader):
    """`segments` file (key wav-key begin end) over a wav.scp (data_handler.py:416-436)."""

    def __init__(self, wav_scp, segments, sr=None, normalize=True):
        super().__init__(segments, num_tokens=4,
                         value_processor=lambda x: {"wav": x[0], "beg": float(x[1]), "end": float(x[2])})
        self.wav_reader = WaveReader(wav_scp, sr=sr, normalize=normalize)

    def _load(self, key):
        info = self.index_dict[key]
        return self.wav_reader.read(info["wav"], beg=int(info["beg"]), end=int(info["end"]))


class PickleReader(ScpReader):
    """key -> pickle.load(path) (data_handler.py:451-462)."""

    def _load(self, key):
        import pickle
        with open(self.index_dict[key], "rb") as f:
            return pickle.load(f)


class MatReader(ScpReader):
    """key -> scipy.io.loadmat(path)[name] (data_handler.py:465-480)."""

    def __init__(self, mat_scp, key):
        super().__init__(mat_scp)
        self.key = key

    def _load(self, key):
        import scipy.io as sio
        mat_dict = sio.loadmat(self.index_dict[key])
        if self.key not in mat_dict:
            raise KeyError(f"Could not find \'{self.key}\' in python dictionary")
        return mat_dict[self.key]


class BinaryReader(ScpReader):
    """key -> numpy.fromfile(path, dtype), optionally of a fixed length (data_handler.py:538-561)."""

    _TYPES = {"float32": np.float32, "float64": np.float64, "int32": np.int32, "int64": np.int64}

    def __init__(self, bin_scp, length=None, data_type="float32"):
        super().__init__(bin_scp)
        if data_type not in self._TYPES:
            raise RuntimeError(f"Unsupported data type: {data_type}")
        self.fmt = self._TYPES[data_type]
        self.length = length

    def _load(self, key):
        obj = np.fromfile(self.index_dict[key], dtype=self.fmt)
        if self.length is not None and obj.size != self.length:
            raise RuntimeError(f"Expect length {self.length:d}, but got {obj.size:d}")
        return obj


class MatWriter(Writer):
    """<dump_dir>/<key>.mat with the array under "data" (data_handler.py:624-637)."""

    def __init__(self, dump_dir, scp_path=None):
        super().__init__(dump_dir, scp_path, is_dir=True)

    def write(self, key, obj):
        import scipy.io as sio
        self.check_args(obj)
        target = self.path_or_dir / f"{key}.mat"
        sio.savemat(target, {"data": obj})
        self._record(key, target)
