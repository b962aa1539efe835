"""Minimal HDF5 reader (and fixture writer) for the two files the reference dataloader opens:
`visdial_data.h5` (uint32 token matrices written by `h5py.File(...).create_dataset(name, dtype='uint32', data=...)`,
/root/reference/data/prepro.py:264-277) and `data_img.h5` (float features written by torch-hdf5,
data/prepro_img_vgg16.lua) — read by `hdf5.open(path, 'r'):read(name):all()` in dataloader.lua:37-129.

Neither h5py nor libhdf5 exists in this image, so this restates the published HDF5 File Format Specification
(version 2.0) for the "earliest" on-disk structures both writers produce by default:
superblock v0/v1, version-1 object headers (with continuation blocks), old-style groups (symbol-table message ->
v1 B-tree of type 0 + local heap + SNOD symbol nodes, nested groups included), dataspace v1/v2, fixed-point and
IEEE floating-point datatypes of either byte order, and the contiguous / compact / chunked (v1 B-tree of type 1,
optional shuffle + deflate filters) data layouts.  Anything newer (superblock v2/v3, "OHDR" headers, fractal-heap
groups) raises H5Error rather than guessing.

PARITY UNPINNED: there is no HDF5 library here to produce or check a file; `write()` below emits the same structures
for fixtures and `tests/test_h5lite.py` checks the reader against bytes assembled by hand from the specification and
against `write()` round trips.  Reading a real `visdial_data.h5` has not been possible in this environment.
"""
from __future__ import annotations

import mmap
import struct
import zlib
from typing import Dict, List, Optional, Tuple

import numpy as np

SIG = b"\x89HDF\r\n\x1a\n"
UNDEF = 0xFFFFFFFFFFFFFFFF


class H5Error(ValueError):
    pass


# ====================================================================================================== reader
class _Reader:
    def __init__(self, buf, path: Optional[str] = None):
        """`buf`: the file's bytes (bytes or a read-only mmap).  With `path`, contiguous uncompressed native-order datasets
        come back as read-only np.memmap views of the file instead of copies."""
        self.b = buf
        self.path = path
        base = 0
        while base < len(buf) and buf[base:base + 8] != SIG:      # the superblock may sit at 0, 512, 1024, ...
            base = 512 if base == 0 else base * 2
        if base >= len(buf):
            raise H5Error("not an HDF5 file (signature not found)")
        ver = buf[base + 8]
        if ver not in (0, 1):
            raise H5Error("superblock version %d is not supported (only the 'earliest' format, v0/v1)" % ver)
        self.O, self.L = buf[base + 13], buf[base + 14]
        if self.O != 8 or self.L != 8:
            raise H5Error("only 8-byte offsets / lengths are supported")
        p = base + 24 + (4 if ver == 1 else 0)
        self.base_addr = self.u64(p)
        p += 4 * 8                                                 # base, free-space, end-of-file, driver-info addresses
        self.root = self._ste(p)

    # ---- primitives
    def u8(self, p): return self.b[p]
    def u16(self, p): return struct.unpack_from("<H", self.b, p)[0]
    def u32(self, p): return struct.unpack_from("<I", self.b, p)[0]
    def u64(self, p): return struct.unpack_from("<Q", self.b, p)[0]

    def _ste(self, p) -> Tuple[int, int]:
        """symbol table entry -> (link name offset, object header address)"""
        return self.u64(p), self.u64(p + 8)

    def _cstr(self, p) -> str:
        e = self.b.find(b"\x00", p)
        if e < 0:
            raise H5Error("unterminated name in the local heap")
        return self.b[p:e].decode("utf-8")

    # ---- object headers
    def messages(self, addr: int) -> List[Tuple[int, int, int]]:
        """[(type, data offset, data size)] of a version-1 object header, following continuation blocks"""
        a = addr + self.base_addr
        if self.b[a:a + 4] == b"OHDR":
            raise H5Error("version-2 object headers are not supported")
        if self.u8(a) != 1:
            raise H5Error("object header version %d is not supported" % self.u8(a))
        nmsg, size = self.u16(a + 2), self.u32(a + 8)
        blocks = [(a + 16, size)]
        out = []
        while blocks and len(out) < nmsg:
            p, left = blocks.pop(0)
            end = p + left
            while p + 8 <= end and len(out) < nmsg:
                t, sz = self.u16(p), self.u16(p + 2)
                d = p + 8
                out.append((t, d, sz))
                if t == 0x0010:                                    # continuation: offset, length
                    blocks.append((self.u64(d) + self.base_addr, self.u64(d + 8)))
                p = d + sz
        return out

    # ---- groups (old style)
    def _heap_data(self, addr: int) -> int:
        a = addr + self.base_addr
        if self.b[a:a + 4] != b"HEAP":
            raise H5Error("local heap signature missing")
        return self.u64(a + 24) + self.base_addr

    def _group_entries(self, btree: int, heap: int) -> List[Tuple[str, int]]:
        names = self._heap_data(heap)
        out: List[Tuple[str, int]] = []

        def walk(addr):
            a = addr + self.base_addr
            if self.b[a:a + 4] != b"TREE" or self.u8(a + 4) != 0:
                raise H5Error("group B-tree node expected")
            level, used = self.u8(a + 5), self.u16(a + 6)
            p = a + 24
            for i in range(used):
                child = self.u64(p + 8 + i * 16)                  # key_i (8), child_i (8), key_{i+1} ...
                if level > 0:
                    walk(child)
                else:
                    s = child + self.base_addr
                    if self.b[s:s + 4] != b"SNOD":
                        raise H5Error("symbol table node expected")
                    for j in range(self.u16(s + 6)):
                        e = s + 8 + j * 40
                        off, hdr = self._ste(e)
                        out.append((self._cstr(names + off), hdr))
        walk(btree)
        return out

    def walk(self) -> Dict[str, int]:
        """every dataset of the file: 'path/name' -> object header address"""
        found: Dict[str, int] = {}

        def visit(hdr: int, prefix: str, depth: int):
            if depth > 16:
                raise H5Error("group nesting too deep (cycle?)")
            msgs = self.messages(hdr)
            st = [m for m in msgs if m[0] == 0x0011]
            if st:
                d = st[0][1]
                for name, child in self._group_entries(self.u64(d), self.u64(d + 8)):
                    visit(child, prefix + name + "/", depth + 1)
            elif any(m[0] == 0x0008 for m in msgs):
                found[prefix.rstrip("/")] = hdr
        visit(self.root[1], "", 0)
        return found

    # ---- datasets
    def _dtype(self, d: int) -> np.dtype:
        cls, bits0, size = self.u8(d) & 0x0F, self.u8(d + 1), self.u32(d + 4)
        order = ">" if bits0 & 1 else "<"
        if cls == 0:
            kind = "i" if bits0 & 0x08 else "u"
            if size not in (1, 2, 4, 8):
                raise H5Error("integer size %d" % size)
            return np.dtype("%s%s%d" % (order, kind, size))
        if cls == 1:
            if size not in (2, 4, 8):
                raise H5Error("float size %d" % size)
            return np.dtype("%sf%d" % (order, size))
        raise H5Error("datatype class %d is not supported (only integers and IEEE floats)" % cls)

    def _shape(self, d: int) -> Tuple[int, ...]:
        ver, rank = self.u8(d), self.u8(d + 1)
        p = d + (8 if ver == 1 else 4)
        if ver not in (1, 2):
            raise H5Error("dataspace version %d" % ver)
        return tuple(self.u64(p + 8 * i) for i in range(rank))

    def _filters(self, d: int) -> List[Tuple[int, List[int]]]:
        ver, n = self.u8(d), self.u8(d + 1)
        p = d + (8 if ver == 1 else 2)
        out = []
        for _ in range(n):
            fid = self.u16(p)
            if ver == 1 or fid >= 256:
                nlen = self.u16(p + 2); p += 4
            else:
                nlen = 0; p += 2
            ncd = self.u16(p + 2); p += 4                         # flags (2), number of client values (2)
            p += (nlen + 7) // 8 * 8 if ver == 1 else nlen
            cd = [self.u32(p + 4 * i) for i in range(ncd)]
            p += 4 * ncd + (4 if (ver == 1 and ncd % 2) else 0)
            out.append((fid, cd))
        return out

    def read(self, hdr: int) -> np.ndarray:
        msgs = {t: (d, sz) for t, d, sz in self.messages(hdr)}
        if 0x0001 not in msgs or 0x0003 not in msgs or 0x0008 not in msgs:
            raise H5Error("object is not a simple dataset")
        shape, dt = self._shape(msgs[0x0001][0]), self._dtype(msgs[0x0003][0])
        n = int(np.prod(shape)) if shape else 1
        d = msgs[0x0008][0]
        ver = self.u8(d)
        if ver == 3:
            cls = self.u8(d + 1)
            if cls == 1:                                           # contiguous
                addr, size = self.u64(d + 2), self.u64(d + 10)
                if addr == UNDEF:
                    return np.zeros(shape, dt.newbyteorder("="))
                return self._contiguous(addr, shape, dt, n)
            elif cls == 0:                                         # compact
                size = self.u16(d + 2)
                raw = self.b[d + 4: d + 4 + size]
            elif cls == 2:
                rank = self.u8(d + 2)
                bt = self.u64(d + 3)
                cdims = [self.u32(d + 11 + 4 * i) for i in range(rank)]
                filters = self._filters(msgs[0x000B][0]) if 0x000B in msgs else []
                return self._chunked(bt, shape, dt, cdims[:-1], filters)
            else:
                raise H5Error("layout class %d" % cls)
        elif ver in (1, 2):
            rank, cls = self.u8(d + 1), self.u8(d + 2)
            if cls != 1:
                raise H5Error("layout version %d: only contiguous storage is supported" % ver)
            return self._contiguous(self.u64(d + 8), shape, dt, n)
        else:
            raise H5Error("data layout version %d is not supported" % ver)
        return self._decode(raw, shape, dt, n)

    @staticmethod
    def _decode(raw, shape, dt: np.dtype, n: int) -> np.ndarray:
        if len(raw) < n * dt.itemsize:
            raise H5Error("dataset data truncated")
        return np.frombuffer(raw, dtype=dt, count=n).reshape(shape).astype(dt.newbyteorder("="))

    def _contiguous(self, addr: int, shape, dt: np.dtype, n: int) -> np.ndarray:
        """A contiguous dataset: a read-only memmap at its data offset when it is already in native byte order (no host
        copy of a multi-GB feature file), else a decoded copy."""
        start = addr + self.base_addr
        native = dt == dt.newbyteorder("=")
        if self.path is None or not native or not shape or n == 0:
            return self._decode(self.b[start:start + n * dt.itemsize], shape, dt, n)
        if start + n * dt.itemsize > len(self.b):
            raise H5Error("dataset data truncated")
        return np.memmap(self.path, dtype=dt.newbyteorder("="), mode="r", offset=start, shape=tuple(shape))

    def _chunked(self, btree: int, shape, dt: np.dtype, cdims: List[int], filters) -> np.ndarray:
        if btree == UNDEF:
            return np.zeros(shape, dt.newbyteorder("="))
        rank = len(shape)
        out = np.zeros(shape, dt.newbyteorder("="))
        keysz = 8 + 8 * (rank + 1)

        def walk(addr):
            a = addr + self.base_addr
            if self.b[a:a + 4] != b"TREE" or self.u8(a + 4) != 1:
                raise H5Error("chunk B-tree node expected")
            level, used = self.u8(a + 5), self.u16(a + 6)
            p = a + 24
            for i in range(used):
                k = p + i * (keysz + 8)
                nbytes, mask = self.u32(k), self.u32(k + 4)
                offs = [self.u64(k + 8 + 8 * j) for j in range(rank)]
                child = self.u64(k + keysz)
                if level > 0:
                    walk(child)
                    continue
                raw = self.b[child + self.base_addr: child + self.base_addr + nbytes]
                for idx in range(len(filters) - 1, -1, -1):       # undo the pipeline in reverse order
                    if mask & (1 << idx):
                        continue
                    fid, cd = filters[idx]
                    if fid == 1:
                        raw = zlib.decompress(raw)
                    elif fid == 2:                                 # shuffle
                        es = cd[0] if cd else dt.itemsize
                        raw = np.frombuffer(raw, np.uint8).reshape(es, -1).T.tobytes()
                    else:
                        raise H5Error("filter %d is not supported" % fid)
                chunk = np.frombuffer(raw, dtype=dt, count=int(np.prod(cdims))).reshape(cdims)
                sl = tuple(slice(o, min(o + c, s)) for o, c, s in zip(offs, cdims, shape))
                out[sl] = chunk[tuple(slice(0, s.stop - s.start) for s in sl)]
        walk(btree)
        return out


def read(path: str, names: Optional[List[str]] = None) -> Dict[str, np.ndarray]:
    """All (or the named) datasets of an HDF5 file as native-endian numpy arrays: the `file:read(name):all()` of
    dataloader.lua:45-129.  Contiguous, uncompressed, native-byte-order datasets are read-only np.memmap views of the file
    (pages are read when touched); chunked, filtered, compact and byte-swapped ones are decoded into new arrays."""
    with open(path, "rb") as f:
        try:
            buf = mmap.mmap(f.fileno(), 0, access=mmap.ACCESS_READ)
        except ValueError:                                         # an empty file cannot be mapped
            raise H5Error("not an HDF5 file (empty)")
    with buf:
        r = _Reader(buf, path)
        table = r.walk()
        if names is not None:
            missing = [n for n in names if n.lstrip("/") not in table]
            if missing:
                raise H5Error("datasets not in file: %s" % ", ".join(missing))
            table = {n.lstrip("/"): table[n.lstrip("/")] for n in names}
        return {k: r.read(v) for k, v in table.items()}


def split(datasets: Dict[str, np.ndarray], dtype: str) -> Dict[str, np.ndarray]:
    """`{'ques_train': .., 'ques_length_train': .., ...}` -> the per-split dict visdial_b200.dataloader takes
    (dataset names without the `_<dtype>` suffix; `images_<dtype>` of the image file becomes `images`)."""
    suf = "_" + dtype
    return {k[:-len(suf)]: v for k, v in datasets.items() if k.endswith(suf)}


# ====================================================================================================== fixture writer
def _pad8(b: bytes) -> bytes:
    return b + b"\x00" * (-len(b) % 8)


def _msg(t: int, data: bytes) -> bytes:
    data = _pad8(data)
    return struct.pack("<HHB3x", t, len(data), 0) + data


def _ohdr(msgs: List[bytes]) -> bytes:
    body = b"".join(msgs)
    return struct.pack("<BxHII4x", 1, len(msgs), 1, len(body)) + body


def _dtype_msg(dt: np.dtype) -> bytes:
    if dt.kind in "iu":
        bits = (0x08 if dt.kind == "i" else 0)
        return struct.pack("<BBBBI", 0x10, bits, 0, 0, dt.itemsize) + struct.pack("<HH", 0, 8 * dt.itemsize)
    if dt.kind == "f" and dt.itemsize in (4, 8):
        e, m, bias = (8, 23, 127) if dt.itemsize == 4 else (11, 52, 1023)
        return struct.pack("<BBBBI", 0x11, 0x20, 8 * dt.itemsize - 1, 0, dt.itemsize) + \
            struct.pack("<HHBBBBI", 0, 8 * dt.itemsize, m, e, 0, m, bias)
    raise H5Error("cannot write dtype %s" % dt)


def write(path: str, datasets: Dict[str, np.ndarray], chunks: Optional[Dict[str, Tuple[int, ...]]] = None,
          gzip: bool = False):
    """Fixture writer: superblock v0, one old-style root group, contiguous datasets (or chunked [+ deflate] for the
    names in `chunks`).  Emits the structures the reader expects from h5py / torch-hdf5 defaults; it is NOT claimed to
    be accepted by libhdf5 (nothing here can check that)."""
    chunks = chunks or {}
    names = sorted(datasets)
    if len(names) > 8 * 32:
        raise H5Error("fixture writer: at most 256 datasets")
    leaf_k, internal_k, chunk_k = 4, 16, 32
    pos = 96                                                       # superblock size (v0, 8-byte offsets)
    blobs: List[Tuple[int, bytes]] = []

    def put(b: bytes) -> int:
        nonlocal pos
        addr = pos
        blobs.append((addr, b))
        pos += len(b) + (-len(b) % 8)
        return addr

    # local heap data: offset 0 = empty string (the root's own name), then the dataset names
    heap = bytearray(b"\x00" * 8)
    name_off = {}
    for n in names:
        name_off[n] = len(heap)
        heap += _pad8(n.encode() + b"\x00")
    hdr_addr = {}
    for n in names:
        a = np.ascontiguousarray(datasets[n])
        dt = a.dtype.newbyteorder("<") if a.dtype.byteorder == ">" else a.dtype
        a = a.astype(dt, copy=False)
        space = struct.pack("<BBB5x", 1, a.ndim, 0) + b"".join(struct.pack("<Q", s) for s in a.shape)
        msgs = [_msg(0x0001, space), _msg(0x0003, _dtype_msg(np.dtype(dt)))]
        if n in chunks:
            cd = tuple(chunks[n])
            grid = [range(0, s, c) for s, c in zip(a.shape, cd)]
            entries = []
            for offs in np.ndindex(*[len(g) for g in grid]):
                o = [g[i] for g, i in zip(grid, offs)]
                chunk = np.zeros(cd, dt)
                sl = tuple(slice(x, min(x + c, s)) for x, c, s in zip(o, cd, a.shape))
                chunk[tuple(slice(0, s.stop - s.start) for s in sl)] = a[sl]
                raw = chunk.tobytes()
                if gzip:
                    raw = zlib.compress(raw, 4)
                entries.append((len(raw), o, put(raw)))
            if len(entries) > 2 * chunk_k:
                raise H5Error("fixture writer: too many chunks for one B-tree node")
            keysz = 8 + 8 * (a.ndim + 1)
            node = b"TREE" + struct.pack("<BBHQQ", 1, 0, len(entries), UNDEF, UNDEF)
            for nbytes, o, addr in entries:
                node += struct.pack("<II", nbytes, 0) + b"".join(struct.pack("<Q", x) for x in o) + struct.pack("<Q", 0)
                node += struct.pack("<Q", addr)
            node += struct.pack("<II", 0, 0) + b"".join(struct.pack("<Q", s) for s in a.shape) + struct.pack("<Q", 0)
            node += b"\x00" * ((2 * chunk_k - len(entries)) * (keysz + 8))
            bt = put(node)
            lay = struct.pack("<BBB", 3, 2, a.ndim + 1) + struct.pack("<Q", bt) + \
                b"".join(struct.pack("<I", c) for c in cd) + struct.pack("<I", dt.itemsize)
            if gzip:
                msgs.append(_msg(0x000B, struct.pack("<BB6x", 1, 1) + struct.pack("<HHHH", 1, 0, 1, 1) + struct.pack("<II", 4, 0)))
        else:
            data_addr = put(a.tobytes()) if a.size else UNDEF
            lay = struct.pack("<BB", 3, 1) + struct.pack("<QQ", data_addr, a.nbytes)
        msgs.append(_msg(0x0008, lay))
        hdr_addr[n] = put(_ohdr(msgs))

    # symbol nodes (2 * leaf_k entries each), one level-0 B-tree node over them
    snods = []
    for i in range(0, max(len(names), 1), 2 * leaf_k):
        part = names[i:i + 2 * leaf_k]
        body = b"SNOD" + struct.pack("<BxH", 1, len(part))
        for n in part:
            body += struct.pack("<QQII16x", name_off[n], hdr_addr[n], 0, 0)
        body += b"\x00" * (40 * (2 * leaf_k - len(part)))
        snods.append((put(body), name_off[part[-1]] if part else 0))
    node = b"TREE" + struct.pack("<BBHQQ", 0, 0, len(snods), UNDEF, UNDEF) + struct.pack("<Q", 0)
    for addr, last in snods:
        node += struct.pack("<QQ", addr, last)
    node += b"\x00" * (16 * (2 * internal_k - len(snods)))
    bt_addr = put(node)
    heap_data = put(bytes(heap))
    heap_addr = put(b"HEAP" + struct.pack("<B3xQQQ", 0, len(heap), UNDEF, heap_data))
    root_hdr = put(_ohdr([_msg(0x0011, struct.pack("<QQ", bt_addr, heap_addr))]))
    sb = SIG + struct.pack("<BBBBBBBBHHI", 0, 0, 0, 0, 0, 8, 8, 0, leaf_k, internal_k, 0)
    sb += struct.pack("<QQQQ", 0, UNDEF, pos, UNDEF)
    sb += struct.pack("<QQII", 0, root_hdr, 1, 0) + struct.pack("<QQ", bt_addr, heap_addr)
    assert len(sb) == 96
    out = bytearray(pos)
    out[0:96] = sb
    for addr, b in blobs:
        out[addr:addr + len(b)] = b
    with open(path, "wb") as f:
        f.write(bytes(out))
