"""A small pure-Python reader (and writer, for tests) of the HDF5 subset that Keras weight files use.

``model.load_weights(path, by_name=True)`` (reference ``ssd300_training.ipynb:162``, ``README.md:223-239``) reads files written
by ``h5py`` with its default ``libver='earliest'``: superblock version 0, "old style" groups (symbol-table message -> version-1
B-tree + local heap + SNOD nodes), version-1 object headers, float datasets with contiguous (or chunked, optionally
gzip / shuffle filtered) layout, and attributes holding fixed-length strings (``layer_names`` / ``weight_names``).  ``h5py`` is
not available offline, so this module implements exactly that subset from the HDF5 File Format Specification (version 2.0,
sections II.A superblock, III.A B-trees, III.B symbol-table nodes, III.D local heaps, IV.A object headers and the messages
0x01 dataspace, 0x03 datatype, 0x08 layout, 0x0B filter pipeline, 0x0C attribute, 0x10 continuation, 0x11 symbol table).
Anything outside the subset (new-style groups, superblock >= 2, variable-length data) raises ``NotImplementedError`` with the
name of the feature, never a silent misread.

``read_datasets(path)`` -> ``{'/group/sub/name': ndarray}``;  ``read_attributes(path, '/')`` -> ``{name: value}`` (fixed-length
strings / numeric arrays only);  ``read_optimizer_weights(path)`` -> ``[(name, array)]`` of ``/optimizer_weights``;
``read_keras_weights(path)`` -> ``{'conv1_1/kernel': ndarray}`` in the file's layer order; ``read_keras_file(path)`` -> the
layers, weights and attributes in the file's order (``KerasFile``).
``write_keras_weights(path, layers)`` writes a file with the same structures (``model.save`` / ``save_weights`` and the tests use
it; files from real h5py use the same structures with different block placement); ``write_keras_file(path, keras_file,
replace=...)`` writes a ``KerasFile`` back with chosen weights replaced (the weight-sampling tutorial's edit)."""
import struct
import zlib

import numpy as np

SIGNATURE = b'\x89HDF\r\n\x1a\n'
UNDEF = 0xFFFFFFFFFFFFFFFF


# =================================================================================================
# reader
# =================================================================================================
class _Reader:
    def __init__(self, buf):
        self.b = buf
        if buf[:8] != SIGNATURE:
            raise ValueError('not an HDF5 file (signature mismatch)')
        ver = buf[8]
        if ver not in (0, 1):
            raise NotImplementedError('HDF5 superblock version %d (files written with libver="latest") is not supported; '
                                      'Keras / h5py write version 0 by default' % ver)
        size_off, size_len = buf[13], buf[14]
        if size_off != 8 or size_len != 8:
            raise NotImplementedError('HDF5 files with %d-byte offsets are not supported' % size_off)
        o = 24 if ver == 0 else 28                      # v1 has 4 extra bytes (indexed-storage K, reserved)
        self.base, _free, self.eof, _drv = struct.unpack_from('<QQQQ', buf, o)
        o += 32
        # root group symbol table entry
        self.root_header = struct.unpack_from('<Q', buf, o + 8)[0]

    # ---- low level -------------------------------------------------------------------------------
    def _messages(self, addr):
        """All (type, flags, payload_offset, size) messages of a version-1 object header, following continuations."""
        b = self.b
        ver = b[addr]
        if ver != 1:
            if b[addr:addr + 4] == b'OHDR':
                raise NotImplementedError('version-2 object headers (libver="latest") are not supported')
            raise ValueError('bad object header version %d at %d' % (ver, addr))
        nmsg = struct.unpack_from('<H', b, addr + 2)[0]
        hsize = struct.unpack_from('<I', b, addr + 8)[0]
        blocks = [(addr + 16, hsize)]                   # 12-byte prefix padded to 16
        out = []
        while blocks and len(out) < nmsg:
            o, size = blocks.pop(0)
            end = o + size
            while o + 8 <= end and len(out) < nmsg:
                mtype, msize, flags = struct.unpack_from('<HHB', b, o)
                body = o + 8
                if mtype == 0x10:                       # continuation
                    co, cl = struct.unpack_from('<QQ', b, body)
                    blocks.append((co, cl))
                out.append((mtype, flags, body, msize))
                o = body + msize
        return out

    def _heap_string(self, heap_addr, off):
        b = self.b
        if b[heap_addr:heap_addr + 4] != b'HEAP':
            raise ValueError('bad local heap signature')
        data_addr = struct.unpack_from('<Q', b, heap_addr + 24)[0]
        s = data_addr + off
        e = s
        while b[e] != 0:
            e += 1
        return bytes(b[s:e]).decode('utf-8')

    def _group_entries(self, btree_addr, heap_addr):
        """(name, object header address) of every link of an old-style group."""
        b = self.b
        out = []

        def walk(addr):
            if b[addr:addr + 4] == b'SNOD':
                n = struct.unpack_from('<H', b, addr + 6)[0]
                for i in range(n):
                    e = addr + 8 + 40 * i
                    name_off, hdr = struct.unpack_from('<QQ', b, e)
                    out.append((self._heap_string(heap_addr, name_off), hdr))
                return
            if b[addr:addr + 4] != b'TREE':
                raise ValueError('bad B-tree node signature at %d' % addr)
            ntype, level, used = struct.unpack_from('<BBH', b, addr + 4)
            if ntype != 0:
                raise ValueError('expected a group B-tree node')
            o = addr + 24                               # signature 4 + type/level/used 4 + two siblings 16
            for i in range(used):
                child = struct.unpack_from('<Q', b, o + 8)[0]    # key_i (8) then child_i (8)
                walk(child)
                o += 16
        walk(btree_addr)
        return out

    # ---- messages --------------------------------------------------------------------------------
    def _dataspace(self, o):
        b = self.b
        ver, rank, flags = b[o], b[o + 1], b[o + 2]
        if ver == 1:
            p = o + 8
        elif ver == 2:
            p = o + 4
        else:
            raise NotImplementedError('dataspace message version %d' % ver)
        return tuple(struct.unpack_from('<%dQ' % rank, b, p)) if rank else ()

    def _datatype(self, o):
        """-> (numpy dtype, total message size of the type)"""
        b = self.b
        cls = b[o] & 0x0F
        bits0 = b[o + 1]
        size = struct.unpack_from('<I', b, o + 4)[0]
        big = bits0 & 1
        if cls == 1:                                    # floating point
            if size not in (2, 4, 8):
                raise NotImplementedError('%d-byte floats' % size)
            return np.dtype(('>' if big else '<') + 'f%d' % size), 8 + 12
        if cls == 0:                                    # fixed point
            signed = (bits0 >> 3) & 1
            return np.dtype(('>' if big else '<') + ('i' if signed else 'u') + '%d' % size), 8 + 4
        if cls == 3:                                    # fixed-length string
            return np.dtype('S%d' % size), 8
        if cls == 9:
            raise NotImplementedError('variable-length data (HDF5 datatype class 9)')
        raise NotImplementedError('HDF5 datatype class %d' % cls)

    def _filters(self, o):
        b = self.b
        ver, n = b[o], b[o + 1]
        p = o + (8 if ver == 1 else 2)
        out = []
        for _ in range(n):
            fid = struct.unpack_from('<H', b, p)[0]
            if ver == 1 or fid >= 256:
                nlen = struct.unpack_from('<H', b, p + 2)[0]
                flags, ncv = struct.unpack_from('<HH', b, p + 4)
                p += 8 + ((nlen + 7) // 8 * 8 if ver == 1 else nlen)
            else:
                flags, ncv = struct.unpack_from('<HH', b, p + 2)
                p += 6
            cvals = struct.unpack_from('<%dI' % ncv, b, p) if ncv else ()
            p += 4 * ncv
            if ver == 1 and ncv % 2:
                p += 4
            out.append((fid, cvals))
        return out

    def _read_chunked(self, btree, chunk_dims, shape, dtype, filters):
        b = self.b
        rank = len(shape)
        out = np.zeros(shape, dtype=dtype)
        esize = dtype.itemsize

        def walk(addr):
            if b[addr:addr + 4] != b'TREE':
                raise ValueError('bad chunk B-tree node')
            ntype, level, used = struct.unpack_from('<BBH', b, addr + 4)
            o = addr + 24
            ksize = 8 + 8 * (rank + 1)
            for i in range(used):
                csize, fmask = struct.unpack_from('<II', b, o)
                offs = struct.unpack_from('<%dQ' % (rank + 1), b, o + 8)[:rank]
                child = struct.unpack_from('<Q', b, o + ksize)[0]
                if level > 0:
                    walk(child)
                else:
                    raw = bytes(b[child:child + csize])
                    for k, (fid, cv) in reversed(list(enumerate(filters))):
                        if fmask & (1 << k):
                            continue
                        if fid == 1:
                            raw = zlib.decompress(raw)
                        elif fid == 2:          # shuffle
                            n = len(raw) // esize
                            raw = np.frombuffer(raw, np.uint8).reshape(esize, n).T.tobytes()
                        elif fid == 3:          # fletcher32 checksum appended
                            raw = raw[:-4]
                        else:
                            raise NotImplementedError('HDF5 filter %d' % fid)
                    chunk = np.frombuffer(raw, dtype=dtype, count=int(np.prod(chunk_dims))).reshape(chunk_dims)
                    sl = tuple(slice(o_, min(o_ + c, s)) for o_, c, s in zip(offs, chunk_dims, shape))
                    out[sl] = chunk[tuple(slice(0, s.stop - s.start) for s in sl)]
                o += ksize + 8
        if btree != UNDEF:
            walk(btree)
        return out

    def _dataset(self, msgs):
        b = self.b
        shape = dtype = layout = None
        filters = []
        for mtype, flags, o, size in msgs:
            if mtype == 0x01:
                shape = self._dataspace(o)
            elif mtype == 0x03:
                dtype, _ = self._datatype(o)
            elif mtype == 0x0B:
                filters = self._filters(o)
            elif mtype == 0x08:
                ver = b[o]
                if ver == 3:
                    cls = b[o + 1]
                    if cls == 0:
                        n = struct.unpack_from('<H', b, o + 2)[0]
                        layout = ('compact', o + 4, n)
                    elif cls == 1:
                        addr, n = struct.unpack_from('<QQ', b, o + 2)
                        layout = ('contiguous', addr, n)
                    elif cls == 2:
                        nd = b[o + 2]
                        bt = struct.unpack_from('<Q', b, o + 3)[0]
                        dims = struct.unpack_from('<%dI' % nd, b, o + 11)
                        layout = ('chunked', bt, dims[:-1])
                    else:
                        raise NotImplementedError('data layout class %d' % cls)
                elif ver in (1, 2):
                    nd, cls = b[o + 1], b[o + 2]
                    p = o + 8
                    addr = None
                    if cls != 0:
                        addr = struct.unpack_from('<Q', b, p)[0]; p += 8
                    dims = struct.unpack_from('<%dI' % nd, b, p); p += 4 * nd
                    if cls == 1:
                        layout = ('contiguous', addr, None)
                    elif cls == 2:
                        layout = ('chunked', addr, dims[:-1])
                    else:
                        n = struct.unpack_from('<I', b, p)[0]
                        layout = ('compact', p + 4, n)
                else:
                    raise NotImplementedError('data layout message version %d' % ver)
        if shape is None or dtype is None or layout is None:
            return None
        count = int(np.prod(shape)) if shape else 1
        if layout[0] == 'chunked':
            return self._read_chunked(layout[1], layout[2], shape, dtype, filters)
        if layout[1] == UNDEF:
            return np.zeros(shape, dtype=dtype)
        return np.frombuffer(b, dtype=dtype, count=count, offset=layout[1]).reshape(shape).copy()

    def _attribute(self, o):
        b = self.b
        ver = b[o]
        if ver == 1:
            nsz, tsz, ssz = struct.unpack_from('<HHH', b, o + 2)
            p = o + 8
            pad = lambda n: (n + 7) // 8 * 8     # noqa: E731
        elif ver in (2, 3):
            nsz, tsz, ssz = struct.unpack_from('<HHH', b, o + 2)
            p = o + (9 if ver == 3 else 8)
            pad = lambda n: n                    # noqa: E731
        else:
            raise NotImplementedError('attribute message version %d' % ver)
        name = bytes(b[p:p + nsz]).split(b'\x00')[0].decode('utf-8'); p += pad(nsz)
        try:
            dtype, _ = self._datatype(p)
        except NotImplementedError:
            return name, None                    # e.g. variable-length strings ('keras_version'): not needed, skipped
        p += pad(tsz)
        shape = self._dataspace(p) if ssz >= 8 or ver != 1 else ()
        p += pad(ssz)
        count = int(np.prod(shape)) if shape else 1
        val = np.frombuffer(b, dtype=dtype, count=count, offset=p).reshape(shape).copy()
        return name, val

    # ---- traversal ---------------------------------------------------------------------------------
    def walk(self):
        """-> (datasets {path: array}, attributes {group path: {name: value}})"""
        datasets, attrs = {}, {}
        seen = set()

        def visit(addr, path):
            if addr in seen:
                return
            seen.add(addr)
            msgs = self._messages(addr)
            a = {}
            for mtype, flags, o, size in msgs:
                if mtype == 0x0C:
                    n, v = self._attribute(o)
                    if v is not None:
                        a[n] = v
                elif mtype in (0x02, 0x06):
                    raise NotImplementedError('new-style groups (link messages; libver="latest") are not supported')
            attrs[path or '/'] = a
            st = [m for m in msgs if m[0] == 0x11]
            if st:
                bt, heap = struct.unpack_from('<QQ', self.b, st[0][2])
                for name, hdr in self._group_entries(bt, heap):
                    visit(hdr, path + '/' + name)
            else:
                d = self._dataset(msgs)
                if d is not None:
                    datasets[path] = d
        visit(self.root_header, '')
        return datasets, attrs


def read_datasets(path):
    with open(path, 'rb') as f:
        buf = f.read()
    return _Reader(buf).walk()[0]


def read_attributes(path, group='/'):
    with open(path, 'rb') as f:
        buf = f.read()
    return _Reader(buf).walk()[1].get(group, {})


def keras_weight_key(layer, stored_name):
    """The package's name of a weight (``'conv1_1/kernel'``) from its layer and its name in ``weight_names``
    (``'conv1_1/kernel:0'``).  The ``:0`` suffix is removed; Keras-1-style names (``<layer>_W:0`` / ``<layer>_b:0``) are mapped to
    ``kernel`` / ``bias``."""
    name = stored_name.split(':')[0]
    if not name.startswith(layer + '/'):
        leaf = name.split('/')[-1]
        if leaf.startswith(layer + '_'):
            leaf = {'W': 'kernel', 'b': 'bias'}.get(leaf[len(layer) + 1:], leaf[len(layer) + 1:])
        name = layer + '/' + leaf
    return name


def _names(value):
    return [bytes(n).decode('utf-8') for n in np.atleast_1d(value)] if value is not None else []


def _in_listed_order(listed, present):
    """The members of ``present`` (in its order) with those in ``listed`` first, in that order."""
    first = [n for n in listed if n in present]
    seen = set(first)
    return first + [n for n in present if n not in seen]


def _optimizer_weights(datasets, attrs, path):
    names = attrs.get('/optimizer_weights', {}).get('weight_names')
    if names is None:
        return []
    out = []
    for n in _names(names):
        if '/optimizer_weights/' + n not in datasets:
            raise ValueError('%s: optimizer weight %s is listed in weight_names but not stored' % (path, n))
        out.append((n, datasets['/optimizer_weights/' + n]))
    return out


class KerasFile:
    """The contents of a Keras HDF5 weights file or of a full-model file's ``/model_weights``, in the file's own order.

    ``layers``: ``[(layer, attributes, [(stored name, array), ...]), ...]`` in ``layer_names`` order, each layer's weights in
    its ``weight_names`` order (stored names such as ``'conv1_1/kernel:0'``), layers without weights included; groups or
    datasets the attributes do not list follow the listed ones.  ``attrs``: the attributes of the group holding the layers
    (``layer_names``, ``backend``, ``keras_version``).  ``root_attrs``: a full-model file's root attributes (``model_config``,
    ``training_config``, ...); ``{}`` for a weights file, whose root is the layer group.  ``optimizer_weights``: a full-model
    file's ``/optimizer_weights`` as ``[(name, array), ...]``.  Attributes this reader cannot decode (variable-length strings)
    are not kept."""

    def __init__(self, layers, attrs, root_attrs=None, full_model=False, optimizer_weights=()):
        self.layers, self.attrs = layers, attrs
        self.root_attrs, self.full_model, self.optimizer_weights = dict(root_attrs or {}), full_model, list(optimizer_weights)

    def weights(self):
        """``{'conv1_1/kernel': array, ...}`` in layer and weight order (``read_keras_weights``)."""
        return {keras_weight_key(layer, n): np.ascontiguousarray(a) for layer, _, items in self.layers for n, a in items}


def read_keras_file(path):
    """-> ``KerasFile``: the layers, weights and attributes of a Keras weights file (``/<layer>/<layer>/kernel:0``,
    ``model.save_weights``) or of a full-model file (``/model_weights/...``, ``model.save``), in the file's order."""
    with open(path, 'rb') as f:
        datasets, attrs = _Reader(f.read()).walk()
    full = '/model_weights' in attrs and '/model_weights' not in datasets
    top = '/model_weights' if full else ''
    groups = [p[len(top) + 1:] for p in attrs if p not in datasets and p.startswith(top + '/') and '/' not in p[len(top) + 1:]]
    groups = [g for g in groups if g]
    top_attrs = attrs.get(top or '/', {})
    layers = []
    for layer in _in_listed_order(_names(top_attrs.get('layer_names')), groups):
        g = top + '/' + layer
        stored = {p[len(g) + 1:]: a for p, a in datasets.items() if p.startswith(g + '/')}
        gattrs = attrs[g]
        layers.append((layer, gattrs, [(n, stored[n]) for n in _in_listed_order(_names(gattrs.get('weight_names')), list(stored))]))
    return KerasFile(layers, top_attrs, attrs.get('/', {}) if full else {}, full, _optimizer_weights(datasets, attrs, path) if full else ())


def read_keras_weights(path):
    """Keras weight names -> arrays: ``{'conv1_1/kernel': ..., 'conv1_1/bias': ..., 'conv4_3_norm/gamma': ...}``, in the
    file's ``layer_names`` / ``weight_names`` order.

    Handles both layouts Keras writes: a weights file (``/<layer>/<layer>/kernel:0``, ``model.save_weights``) and a full model
    file (``/model_weights/<layer>/<layer>/kernel:0``, ``model.save``).  The names are ``keras_weight_key``'s."""
    return read_keras_file(path).weights()


# =================================================================================================
# writer (model.save / save_weights, rewrites of a read file, test fixtures): superblock v0, old-style groups, v1 object
# headers, contiguous or chunked datasets, fixed-length string attributes -- the same structures h5py's default writes
# =================================================================================================
def _little_endian(a):
    """The writer's datatype messages say little endian; a big-endian array read from another file is converted."""
    return a.astype(a.dtype.newbyteorder('<')) if a.dtype.byteorder == '>' else a


class _Writer:
    def __init__(self):
        self.buf = bytearray(b'\x00' * 96)              # superblock v0 = 56 bytes + 40-byte root symbol table entry

    def _alloc(self, n, align=8):
        while len(self.buf) % align:
            self.buf.append(0)
        o = len(self.buf)
        self.buf.extend(b'\x00' * n)
        return o

    @staticmethod
    def _msg(mtype, body, flags=0):
        body = body + b'\x00' * (-len(body) % 8)
        return struct.pack('<HHB3x', mtype, len(body), flags) + body

    def _header(self, messages):
        body = b''.join(messages)
        o = self._alloc(16 + len(body))
        struct.pack_into('<BxHII4x', self.buf, o, 1, len(messages), 1, len(body))
        self.buf[o + 16:o + 16 + len(body)] = body
        return o

    @staticmethod
    def _dtype_msg(dt):
        dt = np.dtype(dt)
        if dt.kind == 'f':
            prec = dt.itemsize * 8
            exp_size, exp_loc, man_size, bias = {4: (8, 23, 23, 127), 8: (11, 52, 52, 1023), 2: (5, 10, 10, 15)}[dt.itemsize]
            # class 1 v1; bit field: little endian, mantissa normalisation 2 (implied msb), sign location = prec-1
            return struct.pack('<BBBBI', 0x11, 0x20, prec - 1, 0, dt.itemsize) + struct.pack('<HHBBBBI', 0, prec, exp_loc, exp_size, 0, man_size, bias)
        if dt.kind in 'iu':
            return struct.pack('<BBBBI', 0x10, 0x08 if dt.kind == 'i' else 0, 0, 0, dt.itemsize) + struct.pack('<HH', 0, dt.itemsize * 8)
        if dt.kind == 'S':
            return struct.pack('<BBBBI', 0x13, 0x00, 0, 0, dt.itemsize)      # null-terminated ASCII
        raise NotImplementedError(dt)

    @staticmethod
    def _space_msg(shape):
        return struct.pack('<BBB5x', 1, len(shape), 0) + b''.join(struct.pack('<Q', int(s)) for s in shape)

    def _attr_msg(self, name, value):
        value = _little_endian(np.asarray(value))
        nm = name.encode() + b'\x00'
        t, s = self._dtype_msg(value.dtype), self._space_msg(value.shape)
        pad = lambda x: x + b'\x00' * (-len(x) % 8)      # noqa: E731
        return self._msg(0x0C, struct.pack('<BxHHH', 1, len(nm), len(t), len(s)) + pad(nm) + pad(t) + pad(s) + value.tobytes())

    def dataset_chunked(self, arr, chunks, gzip=True, shuffle=True):
        """Chunked layout (one B-tree leaf), optionally shuffle + deflate filtered -- what ``compression='gzip'`` produces."""
        arr = _little_endian(np.ascontiguousarray(arr))
        rank, esize = arr.ndim, arr.dtype.itemsize
        keys = []
        grid = [range(0, s, c) for s, c in zip(arr.shape, chunks)]
        for offs in np.array(np.meshgrid(*grid, indexing='ij')).reshape(rank, -1).T:
            block = np.zeros(chunks, dtype=arr.dtype)
            sl = tuple(slice(int(o), min(int(o) + c, s)) for o, c, s in zip(offs, chunks, arr.shape))
            block[tuple(slice(0, q.stop - q.start) for q in sl)] = arr[sl]
            raw = block.tobytes()
            if shuffle:
                raw = np.frombuffer(raw, np.uint8).reshape(-1, esize).T.tobytes()
            if gzip:
                raw = zlib.compress(raw, 4)
            a = self._alloc(len(raw))
            self.buf[a:a + len(raw)] = raw
            keys.append((len(raw), [int(o) for o in offs], a))
        if len(keys) > 64:
            raise NotImplementedError('more than 64 chunks in the test writer')
        ksize = 8 + 8 * (rank + 1)
        bt = self._alloc(24 + (ksize + 8) * len(keys) + ksize)
        self.buf[bt:bt + 24] = b'TREE' + struct.pack('<BBHQQ', 1, 0, len(keys), UNDEF, UNDEF)
        o = bt + 24
        for size, offs, a in keys:
            struct.pack_into('<II%dQ' % (rank + 1), self.buf, o, size, 0, *(offs + [0])); o += ksize
            struct.pack_into('<Q', self.buf, o, a); o += 8
        struct.pack_into('<II%dQ' % (rank + 1), self.buf, o, 0, 0, *([int(s) for s in arr.shape] + [0]))
        filt = b''
        nf = 0
        if shuffle:
            filt += struct.pack('<HHHH', 2, 0, 1, 1) + struct.pack('<I', esize) + b'\x00' * 4; nf += 1
        if gzip:
            filt += struct.pack('<HHHH', 1, 0, 1, 1) + struct.pack('<I', 4) + b'\x00' * 4; nf += 1
        msgs = [self._msg(0x01, self._space_msg(arr.shape)), self._msg(0x03, self._dtype_msg(arr.dtype), flags=1)]
        if nf:
            msgs.append(self._msg(0x0B, struct.pack('<BB6x', 1, nf) + filt))
        msgs.append(self._msg(0x08, struct.pack('<BBBQ', 3, 2, rank + 1, bt) + b''.join(struct.pack('<I', int(c)) for c in list(chunks) + [esize])))
        return self._header(msgs)

    def dataset(self, arr):
        arr = _little_endian(np.ascontiguousarray(arr).reshape(np.shape(arr)))     # a scalar stays a scalar (Keras' iterations:0)
        data = self._alloc(max(arr.nbytes, 1))
        self.buf[data:data + arr.nbytes] = arr.tobytes()
        layout = struct.pack('<BBQQ', 3, 1, data, arr.nbytes)
        return self._header([self._msg(0x01, self._space_msg(arr.shape)), self._msg(0x03, self._dtype_msg(arr.dtype), flags=1),
                             self._msg(0x08, layout)])

    def group(self, entries, attrs=None):
        """entries: [(name, object header address)] -> object header address of the new group."""
        entries = sorted(entries, key=lambda e: e[0].encode())          # B-tree / SNOD order is by name
        heap_data = bytearray(b'\x00' * 8)                                  # offset 0: the empty string
        name_off = []
        for n, _ in entries:
            name_off.append(len(heap_data))
            heap_data.extend(n.encode() + b'\x00')
            heap_data.extend(b'\x00' * (-len(heap_data) % 8))
        seg = self._alloc(len(heap_data))
        self.buf[seg:seg + len(heap_data)] = heap_data
        heap = self._alloc(32)
        self.buf[heap:heap + 32] = b'HEAP' + struct.pack('<B3xQQQ', 0, len(heap_data), UNDEF, seg)
        # one SNOD per 8 entries (2 * leaf K with K = 4), one level-0 B-tree node on top (internal K = 16 -> 32 children max)
        snods = []
        for i in range(0, max(len(entries), 1), 8):
            part = list(zip(name_off, entries))[i:i + 8]
            node = self._alloc(8 + 40 * 8)
            self.buf[node:node + 8] = b'SNOD' + struct.pack('<BxH', 1, len(part))
            for k, (noff, (n, hdr)) in enumerate(part):
                struct.pack_into('<QQII16x', self.buf, node + 8 + 40 * k, noff, hdr, 0, 0)
            snods.append((node, part[-1][0] if part else 0))
        if len(snods) > 32:
            raise NotImplementedError('more than 256 links per group in the test writer')
        bt = self._alloc(24 + 16 * len(snods) + 8)
        self.buf[bt:bt + 24] = b'TREE' + struct.pack('<BBHQQ', 0, 0, len(snods), UNDEF, UNDEF)
        o = bt + 24
        struct.pack_into('<Q', self.buf, o, 0); o += 8                       # key 0: the empty string
        for node, last_name_off in snods:
            struct.pack_into('<QQ', self.buf, o, node, last_name_off); o += 16
        msgs = [self._msg(0x11, struct.pack('<QQ', bt, heap))]
        for k, v in (attrs or {}).items():
            msgs.append(self._attr_msg(k, v))
        return self._header(msgs), bt, heap

    def finish(self, root_hdr, root_bt, root_heap, path):
        b = self.buf
        b[0:8] = SIGNATURE
        struct.pack_into('<BBBxBBBxHHI', b, 8, 0, 0, 0, 0, 8, 8, 4, 16, 0)
        struct.pack_into('<QQQQ', b, 24, 0, UNDEF, len(b), UNDEF)
        struct.pack_into('<QQII', b, 56, 0, root_hdr, 1, 0)
        struct.pack_into('<QQ', b, 80, root_bt, root_heap)
        with open(path, 'wb') as f:
            f.write(bytes(b))


def read_optimizer_weights(path):
    """The ``/optimizer_weights`` group of a full-model file as ``[(name, array), ...]`` in the order of its ``weight_names``
    attribute (Keras' ``optimizer.get_weights()`` order); ``[]`` when the file has none."""
    with open(path, 'rb') as f:
        datasets, attrs = _Reader(f.read()).walk()
    return _optimizer_weights(datasets, attrs, path)


def _tree(w, items):
    """[('a/b/name', array or object header address), ...] -> the links of one group: datasets for plain names (an address is
    a dataset already written), nested groups for 'a/...' prefixes."""
    links, sub = [], {}
    for name, obj in items:
        head, _, rest = name.partition('/')
        if rest:
            sub.setdefault(head, []).append((rest, obj))
        else:
            links.append((head, obj if isinstance(obj, int) else w.dataset(np.asarray(obj))))
    return links + [(head, w.group(_tree(w, part))[0]) for head, part in sub.items()]


def _write(path, source, chunked=()):
    """``source`` (a ``KerasFile``) -> an HDF5 file: its layers, weights and attributes as given; the weights whose
    ``keras_weight_key`` is in ``chunked`` are stored chunked with shuffle + gzip filters."""
    w = _Writer()
    top = []
    for layer, gattrs, items in source.layers:
        objs = [(n, w.dataset_chunked(a, tuple(max(1, (d + 1) // 2) for d in np.shape(a))) if keras_weight_key(layer, n) in chunked else a)
                for n, a in items]
        top.append((layer, w.group(_tree(w, objs), attrs=gattrs)[0]))
    if source.full_model:
        links = [('model_weights', w.group(top, attrs=source.attrs)[0])]
        if source.optimizer_weights:
            names = np.array([n.encode() for n, _ in source.optimizer_weights])
            links.append(('optimizer_weights', w.group(_tree(w, source.optimizer_weights), attrs={'weight_names': names})[0]))
        root, bt, heap = w.group(links, attrs=source.root_attrs or None)
    else:
        root, bt, heap = w.group(top, attrs=source.attrs)
    w.finish(root, bt, heap, path)


def write_keras_file(path, source, replace=None, include_optimizer=None):
    """Write the ``KerasFile`` ``source`` (``read_keras_file``) to ``path``: the same layers in the same order, the same
    ``weight_names`` and attributes, with the weights named in ``replace`` (``{'conv4_3_norm_mbox_conf/kernel': array, ...}``,
    ``keras_weight_key`` names) stored with the shape and dtype of the new array, and every other dataset as it was.

    A full-model file keeps its ``training_config`` and ``/optimizer_weights`` when nothing is replaced and loses them
    otherwise, since an optimizer state does not fit re-shaped weights; ``include_optimizer=True`` with replaced weights raises
    ``ValueError``, ``include_optimizer=False`` drops them always.  Only the weights file layout and ``/model_weights`` are
    written; other groups of a full-model file are not."""
    replace = dict(replace or {})
    replaced = bool(replace)
    layers = []
    for layer, gattrs, items in source.layers:
        layers.append((layer, gattrs, [(n, replace.pop(keras_weight_key(layer, n), a)) for n, a in items]))
    if replace:
        raise ValueError('%s: no such weights in the source file: %s' % (path, sorted(replace)))
    keep = (not replaced) if include_optimizer is None else bool(include_optimizer)
    if keep and replaced and source.full_model:
        raise ValueError('the training_config and optimizer weights of %s do not fit the replaced weights: write the file with '
                         'include_optimizer=False' % path)
    root_attrs = dict(source.root_attrs)
    if not keep:
        root_attrs.pop('training_config', None)
    _write(path, KerasFile(layers, source.attrs, root_attrs, source.full_model, source.optimizer_weights if keep else ()))


def write_keras_weights(path, weights, full_model=False, chunked=(), root_attrs=None, optimizer_weights=()):
    """``weights``: ``{'conv1_1/kernel': array, 'conv1_1/bias': array, ...}`` -> an HDF5 file with the layout of
    ``model.save_weights`` (``/<layer>/<layer>/kernel:0`` datasets, ``layer_names`` / ``weight_names`` attributes, layers in
    the order of ``weights``); with ``full_model`` everything sits below ``/model_weights`` like in ``model.save``; the weights
    named in ``chunked`` are stored chunked with shuffle + gzip filters; ``root_attrs`` (name -> bytes / array) become
    attributes of the root group, where ``model.save`` keeps ``model_config``.  ``optimizer_weights`` (full model only):
    ``[(name, array), ...]`` stored below ``/optimizer_weights`` -- a name's '/' parts become nested groups -- with their order
    in its ``weight_names`` attribute.  ``write_keras_file`` rewrites a file read with ``read_keras_file`` in its own order."""
    per_layer = {}
    for k, v in weights.items():
        layer, name = k.split('/', 1)
        per_layer.setdefault(layer, []).append((layer + '/' + name + ':0', np.asarray(v)))
    layers = [(layer, {'weight_names': np.array([n.encode() for n, _ in items])}, items) for layer, items in per_layer.items()]
    attrs = {'layer_names': np.array([l.encode() for l in per_layer]), 'backend': np.array(b'tensorflow'), 'keras_version': np.array(b'2.1.4')}
    ra = {k: (np.array(v) if isinstance(v, (bytes, str)) else np.asarray(v)) for k, v in (root_attrs or {}).items()}
    if not full_model:
        if optimizer_weights:
            raise ValueError('optimizer weights belong to a full-model file')
        attrs.update(ra)
        ra = {}
    _write(path, KerasFile(layers, attrs, ra, full_model, optimizer_weights), chunked)
