"""Thin object layer over the C ABI: Engine (one cnhe_ctx) and Vec (one cnhe_vec handle).

This is binding code only -- every method is one call into libcnhe.so.  The reference-shaped API (IFactory, IVector,
IMatrix, layers) lives in he.py / layers.py on top of this."""
import ctypes as C
import sys
import weakref

import numpy as np

from . import _lib
from ._lib import U64P, DBLP, VECP, check

DENSE, SPARSE = 0, 1
ALL_SLOTS = 0x7FFFFFFF


def _u64(a):
    return np.ascontiguousarray(a, dtype=np.uint64)


def _p(a):
    return a.ctypes.data_as(U64P)


def _cuda_tensor(x):
    """True for a torch tensor in CUDA memory (torch is never imported here: a tensor means the caller already has it)."""
    torch = sys.modules.get("torch")
    return torch is not None and isinstance(x, torch.Tensor) and x.is_cuda


def _vec_array(vecs):
    arr = (VECP * len(vecs))()
    for i, v in enumerate(vecs):
        arr[i] = None if v is None else v.h
    return arr


class Vec:
    """Owning handle of a cnhe_vec (== EncryptedSealBfvVector).  Dispose() mirrors IDisposable."""

    __slots__ = ("eng", "h", "_m", "__weakref__")

    def __init__(self, eng, handle):
        self.eng = eng
        self.h = VECP(handle) if not isinstance(handle, VECP) else handle
        self._m = None  # metadata cache: a cnhe_vec is immutable except for RegisterScale / RegisterDim
        eng._live.add(self)

    def dispose(self):
        if self.h:
            if self.eng.h:  # a closed engine has already released every vector
                self.eng.L.cnhe_vec_destroy(self.h)
            self.h = VECP(None)

    def __del__(self):
        try:
            self.dispose()
        except Exception:
            pass

    def meta(self):
        if self._m is not None:
            return self._m
        dim, bs = C.c_uint64(), C.c_uint64()
        scale = C.c_double()
        fmt, enc, blocks = C.c_int(), C.c_int(), C.c_int()
        check(self.eng.L.cnhe_vec_meta(self.h, C.byref(dim), C.byref(scale), C.byref(fmt), C.byref(enc), C.byref(blocks), C.byref(bs)))
        self._m = dict(dim=dim.value, scale=scale.value, format=fmt.value, encrypted=bool(enc.value), blocks=blocks.value, block_size=bs.value)
        return self._m

    dim = property(lambda s: s.meta()["dim"])
    scale = property(lambda s: s.meta()["scale"])
    format = property(lambda s: s.meta()["format"])
    is_encrypted = property(lambda s: s.meta()["encrypted"])
    blocks = property(lambda s: s.meta()["blocks"])

    def register_scale(self, scale):
        check(self.eng.L.cnhe_vec_register_scale(self.h, float(scale)))
        self._m = None

    def register_dim(self, dim):
        check(self.eng.L.cnhe_vec_register_dim(self.h, int(dim)))
        self._m = None

    def export_raw(self, channel=0, block=0):
        out = np.zeros(self.eng.ct_words, np.uint64)
        check(self.eng.L.cnhe_vec_export_raw(self.eng.h, self.h, channel, block, _p(out), out.size))
        return out

    @property
    def key_slot(self):
        """The key slot whose evaluation keys this encrypted vector's key switches use (-1: a plain vector)."""
        s = C.c_int()
        check(self.eng.L.cnhe_vec_key_slot(self.h, C.byref(s)))
        return s.value

    def set_key_slot(self, slot):
        """Bind this encrypted vector to a key slot (a ciphertext uploaded by the client whose keys are in that slot)."""
        check(self.eng.L.cnhe_vec_set_key_slot(self.h, int(slot)))

    def device_ptr(self, channel=0):
        p, w = C.c_uint64(), C.c_size_t()
        check(self.eng.L.cnhe_vec_device_ptr(self.h, channel, C.byref(p), C.byref(w)))
        return p.value, w.value


class Diag:
    """Owning handle of a cnhe_diag: a plain matrix prepared for the diagonal (baby-step / giant-step) product."""

    __slots__ = ("eng", "h", "__weakref__")

    def __init__(self, eng, handle):
        self.eng = eng
        self.h = C.c_void_p(handle) if not isinstance(handle, C.c_void_p) else handle
        eng._live.add(self)

    def dispose(self):
        if self.h:
            if self.eng.h:
                self.eng.L.cnhe_diag_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.dispose()
        except Exception:
            pass

    def info(self):
        """dict(n_rows, dim, n1, n2, n_diags, device_bytes): n1 baby steps, n2 giant steps, the stored (nonzero) diagonals."""
        r, n1, n2, nd = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        dim, nb = C.c_uint64(), C.c_uint64()
        check(self.eng.L.cnhe_diag_info(self.h, C.byref(r), C.byref(dim), C.byref(n1), C.byref(n2), C.byref(nd), C.byref(nb)))
        return dict(n_rows=r.value, dim=dim.value, n1=n1.value, n2=n2.value, n_diags=nd.value, device_bytes=nb.value)

    def fold_width(self):
        """The fold width W of a matrix from Engine.diag_prepare(fold_width=...), 0 for an unfolded one."""
        w = C.c_int()
        check(self.eng.L.cnhe_diag_fold_width(self.h, C.byref(w)))
        return w.value

    def export(self, channel, index):
        """(plaintext coefficients mod t [N], (b, g, h)) of stored diagonal `index` (stored by g, then b, then h)."""
        out = np.zeros(self.eng.N, np.uint64)
        bgh = (C.c_int * 3)()
        check(self.eng.L.cnhe_diag_export(self.eng.h, self.h, int(channel), int(index), _p(out), out.size, bgh))
        return out, (bgh[0], bgh[1], bgh[2])

    def ntt_info(self):
        """dict(giant_steps, diags, bytes): the prefix of giant-step groups held resident in NTT form (Engine.diag_prepare's ntt_bytes), its
        diagonals and the device bytes of their NTT forms over all channels."""
        g, nd, nb = C.c_int(), C.c_int(), C.c_uint64()
        check(self.eng.L.cnhe_diag_ntt_info(self.h, C.byref(g), C.byref(nd), C.byref(nb)))
        return dict(giant_steps=g.value, diags=nd.value, bytes=nb.value)

    def export_ntt(self, channel, index):
        """[k][N] words of resident diagonal `index` of a channel: lifted into every q_l and forward transformed (canonical)."""
        out = np.zeros((len(self.eng.q), self.eng.N), np.uint64)
        check(self.eng.L.cnhe_diag_export_ntt(self.eng.h, self.h, int(channel), int(index), _p(out), out.size))
        return out


class Graph:
    """Owning handle of a cnhe_graph: a recorded chain of calls, replayed by launch() (include/cnhe.h, cnhe_capture_begin)."""

    __slots__ = ("eng", "h", "__weakref__")

    def __init__(self, eng, handle):
        self.eng = eng
        self.h = C.c_void_p(handle) if not isinstance(handle, C.c_void_p) else handle
        eng._live.add(self)

    def launch(self):
        """Enqueue one replay (asynchronous, ordered with the engine's other calls)."""
        check(self.eng.L.cnhe_graph_launch(self.h))

    def slots(self):
        """The graph's key positions: the distinct key slots its recorded key switches read, ascending (include/cnhe.h, cnhe_graph_slots)."""
        n = C.c_int32()
        check(self.eng.L.cnhe_graph_slots(self.h, None, 0, C.byref(n)))
        out = (C.c_int32 * max(n.value, 1))()
        check(self.eng.L.cnhe_graph_slots(self.h, out, n.value, C.byref(n)))
        return list(out[:n.value])

    def bind(self, slots):
        """From the next launch on, key position i (slots()[i]) reads key slot slots[i]'s keys (include/cnhe.h, cnhe_graph_bind)."""
        arr = (C.c_int32 * max(len(slots), 1))(*[int(s) for s in slots])
        check(self.eng.L.cnhe_graph_bind(self.h, arr, len(slots)))

    def info(self):
        """dict(kernel_nodes, device_bytes): the graph's kernel nodes and the device memory it owns."""
        kn, nb = C.c_uint64(), C.c_uint64()
        check(self.eng.L.cnhe_graph_info(self.h, C.byref(kn), C.byref(nb)))
        return dict(kernel_nodes=kn.value, device_bytes=nb.value)

    def dispose(self):
        if self.h:
            if self.eng.h:
                check(self.eng.L.cnhe_graph_destroy(self.h))
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.dispose()
        except Exception:
            pass


class Engine:
    """One cnhe_ctx: parameters, device tables and keys for P plaintext moduli (== EncryptedSealBfvFactory)."""

    def __init__(self, plain_primes, N=0, dbc_relin=10, dbc_galois=20, small_modulus_count=-1, device=0, coeff_moduli=None, archive=None,
                 compact_keys=None):
        """archive: bytes of a key archive (cnhe_keys_save / EncryptedSealBfvEnvironment.Save): parameters and keys come from it.
        compact_keys: bytes of a compact key blob (save_compact_keys): parameters from its header, keys expanded on the GPU."""
        self.L = _lib.lib()
        self._live = weakref.WeakSet()
        h = C.c_void_p()
        if archive is not None and compact_keys is not None:
            raise ValueError("give either archive or compact_keys")
        loaded = archive is not None or compact_keys is not None
        if loaded:
            blob = archive if archive is not None else compact_keys
            load = self.L.cnhe_context_load if archive is not None else self.L.cnhe_context_load_compact
            buf = (C.c_ubyte * len(blob)).from_buffer_copy(blob)
            check(load(buf, len(blob), device, C.byref(h)))
            self.h = h
            P = C.c_int()
            check(self.L.cnhe_context_info(self.h, None, None, C.byref(P), None, None, None))
            pp = np.zeros(P.value, np.uint64)
            check(self.L.cnhe_context_plain_moduli(self.h, _p(pp)))
        else:
            pp = _u64(plain_primes)
        if loaded:
            pass
        elif coeff_moduli is None:
            check(self.L.cnhe_context_create(_p(pp), len(pp), N, dbc_relin, dbc_galois, small_modulus_count, device, C.byref(h)))
        else:
            cm = _u64(coeff_moduli)
            check(self.L.cnhe_context_create_custom(_p(pp), len(pp), N, _p(cm), len(cm), dbc_relin, dbc_galois, device, C.byref(h)))
        self.h = h
        self._describe(pp)

    def _describe(self, pp):
        """Reads the context's parameters into attributes (pp: its plaintext primes)."""
        n, k, P, rd, gd, ge = C.c_uint32(), C.c_int(), C.c_int(), C.c_int(), C.c_int(), C.c_int()
        check(self.L.cnhe_context_info(self.h, C.byref(n), C.byref(k), C.byref(P), C.byref(rd), C.byref(gd), C.byref(ge)))
        self.N, self.k, self.P = n.value, k.value, P.value
        self.relin_digits, self.galois_digits, self.n_galois = rd.value, gd.value, ge.value
        self.ct_words = 2 * self.k * self.N
        q = np.zeros(self.k, np.uint64)
        check(self.L.cnhe_context_coeff_moduli(self.h, _p(q)))
        self.q = [int(x) for x in q]
        self.primes = [int(x) for x in pp]
        cnt = C.c_int()
        check(self.L.cnhe_context_bsk_moduli(self.h, None, C.byref(cnt)))
        b = np.zeros(cnt.value, np.uint64)
        check(self.L.cnhe_context_bsk_moduli(self.h, _p(b), C.byref(cnt)))
        self.bsk = [int(x) for x in b]
        self.kb = cnt.value
        self.plain_mod_id = self.k + self.kb  # NTT table id of plaintext modulus 0

    def close(self):
        if self.h:
            self.L.cnhe_capture_abort(self.h)
            live = list(self._live)  # graphs, vectors and matrices hold device buffers of this context: release them first
            for v in sorted(live, key=lambda o: not isinstance(o, Graph)):
                v.dispose()
            self.L.cnhe_context_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- context / keys
    def set_option(self, name, value):
        check(self.L.cnhe_context_set_option(self.h, name.encode(), int(value)))

    def sync(self):
        check(self.L.cnhe_context_sync(self.h))

    def stream(self, channel=0):
        """cudaStream_t (as an integer) of a channel: wrap it with torch.cuda.ExternalStream to order torch / NCCL work with the library's."""
        s = C.c_uint64()
        check(self.L.cnhe_context_stream(self.h, int(channel), C.byref(s)))
        return s.value

    def join_streams(self):
        check(self.L.cnhe_context_join_streams(self.h))

    def fork_streams(self):
        check(self.L.cnhe_context_fork_streams(self.h))

    def keygen(self, seed=None):
        """seed=None: keys and all later encryption randomness from the OS CSPRNG (production).  An integer seed selects the deterministic
        sampler shared with the CPU oracle -- tests only, the keys are predictable."""
        if seed is None:
            check(self.L.cnhe_keys_generate_secure(self.h))
        else:
            check(self.L.cnhe_keys_generate(self.h, int(seed)))

    OP_NAMES = None

    def op_counts(self, reset=False):
        """Evaluator-level operation counters (the reference's OperationsCount)."""
        n = 14
        a = np.zeros(n, np.uint64)
        check(self.L.cnhe_op_counts(self.h, _p(a), n, int(reset)))
        if Engine.OP_NAMES is None:
            Engine.OP_NAMES = [self.L.cnhe_op_name(i).decode() for i in range(n)]
        return {nm: int(v) for nm, v in zip(Engine.OP_NAMES, a)}

    def trace_noise(self, on=True):
        self.set_option("trace_noise", 1 if on else 0)

    def trace_read(self, clear=True):
        """[(operation name, channel, count, budget of the first output, budgets of its first two inputs (-1 unknown), aux)] since the trace
        was last cleared (see cnhe_trace_read in include/cnhe.h)."""
        n = C.c_size_t()
        check(self.L.cnhe_trace_read(self.h, None, 0, C.byref(n), 0))
        a = np.zeros((max(n.value, 1), 8), np.int32)
        check(self.L.cnhe_trace_read(self.h, a.ctypes.data_as(C.POINTER(C.c_int32)), n.value, C.byref(n), int(clear)))
        self.op_counts()
        return [(Engine.OP_NAMES[r[0]], int(r[1]), int(r[2]), int(r[3]), int(r[4]), int(r[5]), r[6] / 1000.0) for r in a[:n.value]]

    def save_keys(self, with_private_keys=False):
        """The key archive of EncryptedSealBfvEnvironment.Save as bytes."""
        n = C.c_size_t()
        check(self.L.cnhe_keys_save(self.h, int(with_private_keys), None, 0, C.byref(n)))
        buf = (C.c_ubyte * n.value)()
        check(self.L.cnhe_keys_save(self.h, int(with_private_keys), buf, n.value, C.byref(n)))
        return bytes(buf)

    def save_compact_keys(self, public=True, relin=True, galois=None):
        """A freshly generated evaluation-key set as one compact blob (bytes) for a server (cnhe_keys_save_compact): a per-channel ChaCha20
        key for every a and bit-packed b.  galois: None = every standard element, [] = none, else a list of elements.  Needs the secret key;
        this engine's own keys are unchanged."""
        sets = (1 if public else 0) | (2 if relin else 0)
        if galois is None:
            elts, n = None, -1
        else:
            arr = _u64(list(galois))
            elts, n = (_p(arr) if arr.size else None), int(arr.size)
        need = C.c_size_t()
        check(self.L.cnhe_keys_save_compact(self.h, sets, elts, n, None, 0, C.byref(need)))
        buf = (C.c_ubyte * need.value)()
        check(self.L.cnhe_keys_save_compact(self.h, sets, elts, n, buf, need.value, C.byref(need)))
        return bytes(buf)

    def add_client_compact(self, blob):
        """Load another client's compact evaluation keys (save_compact_keys of the client's engine; same parameters) into a new key slot;
        returns the slot number.  Vectors bound to it with Vec.set_key_slot are evaluated under those keys."""
        buf = (C.c_ubyte * len(blob)).from_buffer_copy(blob)
        s = C.c_int()
        check(self.L.cnhe_context_add_client_compact(self.h, buf, len(blob), C.byref(s)))
        return s.value

    def remove_client(self, slot):
        check(self.L.cnhe_context_remove_client(self.h, int(slot)))

    # ---- levels (include/cnhe.h, cnhe_context_derive_level; DESIGN 4.17)
    def derive_level(self, k):
        """A new Engine on the first k coefficient primes of this one, holding the restriction of its keys and of every key slot's.  The
        two engines are independent afterwards; vectors move down with mod_switch."""
        h = C.c_void_p()
        check(self.L.cnhe_context_derive_level(self.h, int(k), C.byref(h)))
        child = Engine.__new__(Engine)
        child.L = self.L
        child._live = weakref.WeakSet()
        child.h = h
        child._describe(np.array(self.primes, np.uint64))
        return child

    def mod_switch(self, vecs, to):
        """The encrypted vectors `vecs` of this engine switched to engine `to` (a level of the same family with fewer primes): every
        ciphertext drops the primes it has beyond to.k.  Outputs keep dimension, scale, format and key slot."""
        n = len(vecs)
        out = (VECP * n)()
        check(self.L.cnhe_vecs_mod_switch(self.h, _vec_array(vecs), n, to.h, out))
        return to._wrap_many(out, n, like=vecs)

    # ---- sanitisation (include/cnhe.h, cnhe_vecs_sanitize; DESIGN 4.18)
    def sanitize_max_bits(self):
        """The widest flood sanitize accepts: floor(log2(q / t)) - 2 for the largest plaintext prime t."""
        q = 1
        for x in self.q:
            q *= x
        return min((q // t).bit_length() - 1 for t in self.primes) - 2

    def sanitize(self, vecs, flood_bits):
        """The encrypted vectors `vecs` (key slots may differ) re-randomised under their slots' public keys, with a uniform flood of
        flood_bits bits in their noise: the results decrypt as the inputs do and reveal nothing else about how they were computed as long
        as flood_bits covers the inputs' noise (DESIGN 4.18).  Outputs keep dimension, scale, format and key slot."""
        n = len(vecs)
        out = (VECP * n)()
        check(self.L.cnhe_vecs_sanitize(self.h, _vec_array(vecs), n, int(flood_bits), out))
        return self._wrap_many(out, n, like=vecs)

    def write_vector(self, vec):
        """EncryptedSealBfvVector.Write: the text form of one vector."""
        n = C.c_size_t()
        check(self.L.cnhe_vec_write(self.h, vec.h, None, 0, C.byref(n)))
        buf = C.create_string_buffer(n.value)
        check(self.L.cnhe_vec_write(self.h, vec.h, buf, n.value, C.byref(n)))
        return buf.raw[: n.value].decode("ascii")

    def read_vector(self, text):
        """EncryptedSealBfvVector.Read; returns (Vec, characters consumed)."""
        raw = text.encode("ascii") if isinstance(text, str) else text
        out, used = VECP(), C.c_size_t()
        check(self.L.cnhe_vec_read(self.h, raw, len(raw), C.byref(out), C.byref(used)))
        return Vec(self, out), used.value

    def galois_elts(self):
        a = np.zeros(self.n_galois, np.uint64)
        check(self.L.cnhe_context_galois_elts(self.h, _p(a)))
        return [int(x) for x in a]

    def _key_words(self, what):
        kN = self.k * self.N
        return {0: kN, 1: 2 * kN, 2: self.relin_digits * 2 * kN, 3: self.galois_digits * 2 * kN, 4: self.relin_digits * 2 * kN * 6 // 8}[what]

    def export_key(self, channel, what, arg=0):
        a = np.zeros(self._key_words(what), np.uint64)
        check(self.L.cnhe_keys_export(self.h, channel, what, int(arg), _p(a), a.size))
        return a

    def import_key(self, channel, what, data, arg=0):
        a = _u64(data).ravel()
        check(self.L.cnhe_keys_import(self.h, channel, what, int(arg), _p(a), a.size))

    def set_seed(self, channel, seed):
        check(self.L.cnhe_keys_set_seed(self.h, channel, int(seed)))

    def launch_count(self):
        return int(self.L.cnhe_kernel_launch_count(self.h))

    # ---- graph recording (include/cnhe.h, cnhe_capture_begin)
    def capture_begin(self, levels=None):
        """From now on the context records its calls into a graph instead of running them.  levels: engines of this one's family with
        fewer primes (derive_level) to enlist: their calls and the mod_switch calls between them go into the same graph
        (include/cnhe.h, cnhe_capture_begin_levels)."""
        if levels is None:
            check(self.L.cnhe_capture_begin(self.h))
            self._capture_levels = []
            return
        arr = (C.c_void_p * max(len(levels), 1))(*[e.h.value for e in levels])
        check(self.L.cnhe_capture_begin_levels(self.h, arr, len(levels)))
        self._capture_levels = list(levels)

    def capture_end(self):
        """The recorded calls as a Graph (launch() replays them).  A graph that spans levels is also released when one of them closes."""
        g = C.c_void_p()
        check(self.L.cnhe_capture_end(self.h, C.byref(g)))
        graph = Graph(self, g)
        for e in self.__dict__.pop("_capture_levels", []):
            e._live.add(graph)
        return graph

    def capture_abort(self):
        check(self.L.cnhe_capture_abort(self.h))

    def vecs_assign(self, dst, src):
        """dst[i] takes src[i]'s ciphertext words (same dimension, blocks, format, scale and key slot): new inputs of a recorded graph."""
        if len(dst) != len(src):
            raise ValueError("dst and src differ in length")
        check(self.L.cnhe_vecs_assign(self.h, _vec_array(dst), _vec_array(src), len(dst)))

    # ---- vectors
    def _new(self, fn, v, scale, fmt):
        a = np.ascontiguousarray(v, dtype=np.float64).ravel()
        out = VECP()
        check(fn(self.h, a.ctypes.data_as(DBLP), a.size, float(scale), fmt, C.byref(out)))
        return Vec(self, out)

    def encrypt(self, v, scale=1.0, fmt=DENSE):
        return self._new(self.L.cnhe_vec_encrypt, v, scale, fmt)

    def plain(self, v, scale=1.0, fmt=DENSE):
        return self._new(self.L.cnhe_vec_plain, v, scale, fmt)

    # ---- values in device memory (DESIGN 4.19): torch work is ordered with the library's channel-0 stream by events, never by a
    # device-wide synchronise
    def _library_stream(self, device):
        import torch
        return torch.cuda.ExternalStream(self.stream(0), device=device)

    def _device_rows(self, rows):
        """A CUDA tensor [n][dim] as contiguous float64 on its device, with the library's stream made to wait for the caller's current
        stream (where the tensor, and its conversion, were queued)."""
        import torch
        if rows.dim() != 2:
            raise ValueError("rows must be [n][dim]")
        t = rows.to(torch.float64).contiguous()
        self._library_stream(t.device).wait_stream(torch.cuda.current_stream(t.device))
        return t  # the encrypt calls return once they have read it

    def encrypt_many(self, rows, scale=1.0):
        """Encrypts the rows [n][dim] of a numpy array or a CUDA torch tensor (float64, or converted on its device) as n dense vectors."""
        if _cuda_tensor(rows):
            t = self._device_rows(rows)
            n, dim = t.shape
            out = (VECP * n)()
            check(self.L.cnhe_vecs_encrypt_device(self.h, t.data_ptr(), n, dim, float(scale), out))
            return [Vec(self, out[i]) for i in range(n)]
        a = np.ascontiguousarray(rows, dtype=np.float64)
        n, dim = a.shape
        out = (VECP * n)()
        check(self.L.cnhe_vecs_encrypt(self.h, a.ctypes.data_as(DBLP), n, dim, float(scale), out))
        return [Vec(self, out[i]) for i in range(n)]

    def decrypt(self, vec):
        out = np.zeros(vec.dim, np.float64)
        check(self.L.cnhe_vec_decrypt(self.h, vec.h, out.ctypes.data_as(DBLP), out.size))
        return out

    def decrypt_residues(self, vec):
        """Per-channel residues [P][dim] of the decryption (DecryptFullPrecision joins them with big integers)."""
        out = np.zeros((self.P, vec.dim), np.uint64)
        check(self.L.cnhe_vec_decrypt_residues(self.h, vec.h, _p(out), out.size))
        return out

    def from_residues(self, residues, scale=1.0, fmt=DENSE, encrypt=True):
        r = _u64(residues).reshape(self.P, -1)
        out = VECP()
        check(self.L.cnhe_vec_from_residues(self.h, _p(r), r.shape[1], float(scale), fmt, int(encrypt), C.byref(out)))
        return Vec(self, out)

    def dispose_many(self, vecs):
        """Release a list of Vec handles with one ABI call."""
        live = [v for v in vecs if v is not None and v.h]
        if live and self.h:
            check(self.L.cnhe_vecs_destroy(_vec_array(live), len(live)))
        for v in live:
            v.h = VECP(None)

    def decrypt_many(self, vecs, device=False):
        """The vectors' values [n][dim] as a numpy array, or with device=True (or a torch device) as a float64 CUDA tensor on the current
        CUDA device: ready for work queued on the caller's current stream afterwards, without a host wait."""
        dim = vecs[0].dim
        if device is not False:
            import torch
            dev = torch.device("cuda", torch.cuda.current_device()) if device is True else torch.device(device)
            out = torch.empty((len(vecs), dim), dtype=torch.float64, device=dev)
            lib = self._library_stream(dev)
            lib.wait_stream(torch.cuda.current_stream(dev))  # the allocation's stream order: the library writes after it
            check(self.L.cnhe_vecs_decrypt_device(self.h, _vec_array(vecs), len(vecs), out.data_ptr(), dim))
            torch.cuda.current_stream(dev).wait_stream(lib)
            return out
        out = np.zeros((len(vecs), dim), np.float64)
        check(self.L.cnhe_vecs_decrypt(self.h, _vec_array(vecs), len(vecs), out.ctypes.data_as(DBLP), dim))
        return out

    def import_raw(self, data, blocks, dim, scale=1.0, fmt=DENSE):
        a = _u64(data).ravel()
        assert a.size == self.P * blocks * self.ct_words
        out = VECP()
        check(self.L.cnhe_vec_import_raw(self.h, _p(a), blocks, int(dim), float(scale), fmt, C.byref(out)))
        return Vec(self, out)

    def import_raw_ptr(self, ptr, blocks, dim, scale=1.0, fmt=DENSE):
        """One vector from raw words at a host OR device address, layout [P][blocks][2kN] (multi-GPU exchanges hand over device buffers)."""
        out = VECP()
        check(self.L.cnhe_vec_import_raw(self.h, C.cast(int(ptr), U64P), int(blocks), int(dim), float(scale), fmt, C.byref(out)))
        return Vec(self, out)

    def import_raw_many(self, host_ptr_or_array, n, blocks, dim, scale=1.0, fmt=DENSE):
        """host layout [P][n][blocks][2kN]; accepts a numpy array or a raw host address (e.g. a pinned torch tensor's data_ptr())."""
        if isinstance(host_ptr_or_array, int):
            src = C.cast(host_ptr_or_array, U64P)
        else:
            a = _u64(host_ptr_or_array).ravel()
            assert a.size == self.P * n * blocks * self.ct_words
            src = _p(a)
        out = (VECP * n)()
        check(self.L.cnhe_vecs_import_raw(self.h, src, n, blocks, int(dim), float(scale), fmt, out))
        return self._wrap_many(out, n)

    def encrypt_compact(self, rows, scale=1.0):
        """Seeded secret-key encryption of n dense vectors (rows [n][dim]) into one compact blob (bytes): bit-packed c0 plus one ChaCha20
        key per plaintext modulus from which import_compact regenerates c1 on the GPU.  Needs the secret key.  rows: a numpy array or a
        CUDA torch tensor, as for encrypt_many."""
        if _cuda_tensor(rows):
            t = self._device_rows(rows)
            fn, src = self.L.cnhe_vecs_encrypt_compact_device, t.data_ptr()
        else:
            t = np.ascontiguousarray(rows, dtype=np.float64)
            fn, src = self.L.cnhe_vecs_encrypt_compact, t.ctypes.data_as(DBLP)
        n, dim = t.shape
        need = C.c_size_t()
        check(fn(self.h, src, n, dim, float(scale), None, 0, C.byref(need)))
        buf = (C.c_ubyte * need.value)()
        check(fn(self.h, src, n, dim, float(scale), buf, need.value, C.byref(need)))
        return bytes(buf)

    def import_compact(self, buf_or_ptr, length=None):
        """The vectors of a compact blob (bytes-like, or a host address with `length`, e.g. a pinned torch tensor's data_ptr()) as ordinary
        encrypted dense vectors; asynchronous like import_raw_many.  Pinned memory must stay unchanged until the vectors are consumed."""
        if isinstance(buf_or_ptr, int):
            if length is None:
                raise ValueError("length is required with a host address")
            src, size = C.c_void_p(buf_or_ptr), int(length)
            head = C.string_at(buf_or_ptr, min(size, 24))
        else:
            mv = memoryview(buf_or_ptr).cast("B")
            size = mv.nbytes if length is None else int(length)
            arr = np.frombuffer(mv, dtype=np.uint8)
            src = C.c_void_p(arr.ctypes.data)
            head = bytes(mv[:24])
        cap = int.from_bytes(head[20:24], "little") if len(head) >= 24 else 0
        out = (VECP * max(cap, 1))()
        n = C.c_int()
        check(self.L.cnhe_vecs_import_compact(self.h, src, size, out, cap, C.byref(n)))
        return self._wrap_many(out, n.value)

    def export_raw_many(self, vecs, host_ptr=None):
        n, blocks = len(vecs), vecs[0].blocks
        words = self.P * n * blocks * self.ct_words
        if host_ptr is None:
            a = np.zeros(words, np.uint64)
            check(self.L.cnhe_vecs_export_raw(self.h, _vec_array(vecs), n, _p(a), words))
            return a.reshape(self.P, n, blocks, self.ct_words)
        check(self.L.cnhe_vecs_export_raw(self.h, _vec_array(vecs), n, C.cast(host_ptr, U64P), words))
        return None

    def export_raw_many_async(self, vecs, host_ptr):
        """Queue the device-to-host copies behind the producing kernels; returns a ticket for export_wait().  `host_ptr`: pinned memory."""
        n, blocks = len(vecs), vecs[0].blocks
        t = C.c_int()
        check(self.L.cnhe_vecs_export_raw_async(self.h, _vec_array(vecs), n, C.cast(host_ptr, U64P), self.P * n * blocks * self.ct_words, C.byref(t)))
        return t.value

    def export_wait(self, ticket):
        check(self.L.cnhe_export_wait(self.h, int(ticket)))

    def dev_copy(self, dst, src, words):
        check(self.L.cnhe_dev_copy(self.h, int(dst), int(src), int(words)))

    def prof_enable(self, on=True):
        check(self.L.cnhe_prof_enable(self.h, int(on)))

    def prof_collect(self):
        names = ["ntt_forward", "ntt_inverse", "behz_elementwise", "keyswitch_mac", "scalar_mac_layer", "other", "sanitize_finish"]
        out = {}
        for i, nm in enumerate(names):
            ms, n, b = C.c_double(), C.c_uint64(), C.c_double()
            check(self.L.cnhe_prof_collect(self.h, i, C.byref(ms), C.byref(n), C.byref(b)))
            out[nm] = dict(ms=ms.value, launches=n.value, bytes=b.value)
        return out

    def copy(self, vec):
        out = VECP()
        check(self.L.cnhe_vec_copy(self.h, vec.h, C.byref(out)))
        return Vec(self, out)

    def noise_budget(self, vec, channel=0, block=0):
        b = C.c_int()
        check(self.L.cnhe_noise_budget(self.h, vec.h, channel, block, C.byref(b)))
        return b.value

    def _bin(self, fn, a, b):
        out = VECP()
        check(fn(self.h, a.h, b.h, C.byref(out)))
        return Vec(self, out)

    def add(self, a, b):
        return self._bin(self.L.cnhe_vec_add, a, b)

    def sub(self, a, b):
        return self._bin(self.L.cnhe_vec_sub, a, b)

    def pointwise_multiply(self, a, b):
        return self._bin(self.L.cnhe_vec_pointwise_multiply, a, b)

    def sum_all_slots(self, a, length=ALL_SLOTS, force_column=-1):
        out = VECP()
        check(self.L.cnhe_vec_sum_all_slots(self.h, a.h, int(length), int(force_column), C.byref(out)))
        return Vec(self, out)

    def dot_product(self, a, b, length=ALL_SLOTS, force_column=-1):
        out = VECP()
        check(self.L.cnhe_vec_dot_product(self.h, a.h, b.h, int(length), int(force_column), C.byref(out)))
        return Vec(self, out)

    def rotate(self, a, amount):
        out = VECP()
        check(self.L.cnhe_vec_rotate(self.h, a.h, int(amount), C.byref(out)))
        return Vec(self, out)

    def rotate_many(self, vecs, amount):
        """rotate() of every vector by the same amount in one pass; their key slots may differ."""
        n = len(vecs)
        out = (VECP * n)()
        check(self.L.cnhe_vecs_rotate(self.h, _vec_array(vecs), n, int(amount), out))
        return self._wrap_many(out, n, like=vecs)

    def duplicate(self, a, count):
        out = VECP()
        check(self.L.cnhe_vec_duplicate(self.h, a.h, int(count), C.byref(out)))
        return Vec(self, out)

    def permute(self, a, selections, shifts, output_dim):
        sh = (C.c_int * len(shifts))(*[int(s) for s in shifts])
        out = VECP()
        check(self.L.cnhe_vec_permute(self.h, a.h, _vec_array(selections), sh, len(shifts), int(output_dim), C.byref(out)))
        return Vec(self, out)

    def interleave(self, vecs, shift):
        out = VECP()
        check(self.L.cnhe_vecs_interleave(self.h, _vec_array(vecs), len(vecs), int(shift), C.byref(out)))
        return Vec(self, out)

    def stack(self, vecs):
        out = VECP()
        check(self.L.cnhe_vecs_stack(self.h, _vec_array(vecs), len(vecs), C.byref(out)))
        return Vec(self, out)

    def stack_many(self, groups):
        """stack(g) for every group g (equal lengths; one per client, their key slots may differ) in one pass."""
        B, n = len(groups), len(groups[0])
        if any(len(g) != n for g in groups):
            raise ValueError("every group must have the same number of vectors")
        out = (VECP * B)()
        check(self.L.cnhe_vecs_stack_batch(self.h, _vec_array([v for g in groups for v in g]), n, B, out))
        return self._wrap_many(out, B, like=[g[0] for g in groups])

    def generate_sparse_of_array(self, vecs):
        out = VECP()
        check(self.L.cnhe_vecs_generate_sparse_of_array(self.h, _vec_array(vecs), len(vecs), C.byref(out)))
        return Vec(self, out)

    def mat_mul_colmajor_sparse(self, cols, sparse):
        out = VECP()
        check(self.L.cnhe_mat_mul_colmajor_sparse(self.h, _vec_array(cols), len(cols), sparse.h, C.byref(out)))
        return Vec(self, out)

    def mat_mul_colmajor_sparse_deferred(self, cols, sparse):
        """mat_mul_colmajor_sparse with encrypted columns and an encrypted sparse vector, one relinearisation per output block: the products
        of each chunk of at most product_sum_terms() columns are summed before one BEHZ floor (cnhe.h, DESIGN.md 4.14)"""
        out = VECP()
        check(self.L.cnhe_mat_mul_colmajor_sparse_deferred(self.h, _vec_array(cols), len(cols), sparse.h, C.byref(out)))
        return Vec(self, out)

    def product_sum_terms(self):
        """K_c: the most products one floor of mat_mul_colmajor_sparse_deferred sums in this context"""
        n = C.c_int()
        check(self.L.cnhe_context_product_sum_terms(self.h, C.byref(n)))
        return n.value

    def mat_mul_rowmajor(self, rows, v, force_dense=False):
        out = VECP()
        check(self.L.cnhe_mat_mul_rowmajor(self.h, _vec_array(rows), len(rows), v.h, int(force_dense), C.byref(out)))
        return Vec(self, out)

    def mat_mul_rowmajor_batch(self, rows, vs, force_dense=False):
        """mat_mul_rowmajor(rows, v, force_dense) for every v in vs in one pass (one input per client; their key slots may differ)."""
        B = len(vs)
        out = (VECP * B)()
        check(self.L.cnhe_mat_mul_rowmajor_batch(self.h, _vec_array(rows), len(rows), _vec_array(vs), B, int(force_dense), out))
        return self._wrap_many(out, B)

    def dot_rows_batch(self, rows, vs, length=ALL_SLOTS):
        """[[dot_product(r, v, length) for r in rows] for v in vs] in one pass (one input per client; their key slots may differ), flattened
        client by client."""
        B, R = len(vs), len(rows)
        out = (VECP * (B * R))()
        check(self.L.cnhe_mat_dot_rows_batch(self.h, _vec_array(rows), R, _vec_array(vs), B, int(length), out))
        return self._wrap_many(out, B * R)

    def duplicate_many(self, vecs, count):
        """duplicate(v, count) for every v (one per client) in one pass."""
        B = len(vecs)
        out = (VECP * B)()
        check(self.L.cnhe_vecs_duplicate_batch(self.h, _vec_array(vecs), B, int(count), out))
        return self._wrap_many(out, B)

    def permute_many(self, vecs, perms, output_dim):
        """[permute(v, sel, shifts, output_dim) for (sel, shifts) in perms] for every v (one per client) in one pass, flattened client by
        client; every permutation has the same number of selections (None entries are skipped)."""
        B, P, S = len(vecs), len(perms), len(perms[0][0])
        if any(len(sel) != S or len(sh) != S for sel, sh in perms):
            raise ValueError("every permutation must have the same number of selections and shifts")
        sh = (C.c_int * (P * S))(*[int(s) for _, shifts in perms for s in shifts])
        out = (VECP * (B * P))()
        check(self.L.cnhe_vecs_permute_batch(self.h, _vec_array(vecs), B, _vec_array([s for sel, _ in perms for s in sel]), sh, P, S, int(output_dim),
                                             out))
        return self._wrap_many(out, B * P)

    def interleave_many(self, groups, shift):
        """interleave(g, shift) for every group g (equal lengths; one per client) in one pass."""
        B, n = len(groups), len(groups[0])
        if any(len(g) != n for g in groups):
            raise ValueError("every group must have the same number of vectors")
        out = (VECP * B)()
        check(self.L.cnhe_vecs_interleave_batch(self.h, _vec_array([v for g in groups for v in g]), n, B, int(shift), out))
        return self._wrap_many(out, B)

    def multiply_plain_many(self, vecs, plain):
        """pointwise_multiply(v, plain) for every encrypted v and one plain dense vector in one pass."""
        n = len(vecs)
        out = (VECP * n)()
        check(self.L.cnhe_vecs_multiply_plain(self.h, _vec_array(vecs), n, plain.h, out))
        return self._wrap_many(out, n)

    def mat_mul_rowmajor_shard(self, rows, v, force_dense, first_row, total_rows):
        out = VECP()
        check(self.L.cnhe_mat_mul_rowmajor_shard(self.h, _vec_array(rows), len(rows), v.h, int(force_dense), int(first_row), int(total_rows), C.byref(out)))
        return Vec(self, out)

    def diag_prepare(self, rows, baby_steps=0, ntt_bytes=0, fold_width=None):
        """The plain row vectors of a matrix (as mat_mul_rowmajor takes them) prepared for mat_mul_diagonal; baby_steps = 0 lets the library
        pick n1.  ntt_bytes: device memory the matrix may spend on holding the longest prefix of whole giant-step groups in NTT form, so
        that mat_mul_diagonal skips their lift and transforms (same outputs); 0 holds none, None (or 2**64 - 1) the whole matrix.  The rows
        may be disposed afterwards.  fold_width: None prepares the generalised diagonals (cnhe_diag_prepare); an int prepares the folded
        product for few rows (cnhe_diag_prepare_folded: at most N/2 rows, a power-of-two fold width in [rows, N/2], 0 lets the library
        choose it), whose outputs are dense of dim len(rows)."""
        out = C.c_void_p()
        if fold_width is not None:
            budget = (1 << 64) - 1 if ntt_bytes is None else int(ntt_bytes)
            if not 0 <= budget < 1 << 64:
                raise ValueError("ntt_bytes must be None or in [0, 2**64)")
            check(self.L.cnhe_diag_prepare_folded(self.h, _vec_array(rows), len(rows), int(fold_width), int(baby_steps), budget, C.byref(out)))
        elif ntt_bytes == 0:
            check(self.L.cnhe_diag_prepare(self.h, _vec_array(rows), len(rows), int(baby_steps), C.byref(out)))
        else:
            budget = (1 << 64) - 1 if ntt_bytes is None else int(ntt_bytes)
            if not 0 <= budget < 1 << 64:
                raise ValueError("ntt_bytes must be None or in [0, 2**64)")
            check(self.L.cnhe_diag_prepare_ntt(self.h, _vec_array(rows), len(rows), int(baby_steps), budget, C.byref(out)))
        return Diag(self, out)

    def mat_mul_diagonal(self, diag, vs):
        """The diagonal product of a prepared matrix with every encrypted vector of vs (one per client; their key slots may differ): each
        output decrypts to mat_mul_rowmajor(rows, v, force_dense=True) (a folded matrix: dense of dim len(rows), slot i row i's sum)."""
        B = len(vs)
        out = (VECP * B)()
        check(self.L.cnhe_mat_mul_diagonal(self.h, diag.h, _vec_array(vs), B, out))
        return self._wrap_many(out, B)

    def layer_conv_dense(self, inputs, gather, weights, bias, M, K):
        g = None
        if gather is not None:
            g = np.ascontiguousarray(gather, dtype=np.int32)
            assert g.size == M * K
        out = (VECP * M)()
        check(self.L.cnhe_layer_conv_dense(
            self.h, _vec_array(inputs), len(inputs), None if g is None else g.ctypes.data_as(C.POINTER(C.c_int32)), _vec_array(weights),
            None if bias is None else _vec_array(bias), M, K, out))
        return self._wrap_many(out, M)

    def layer_activation_conv_dense(self, inputs, a, b, c, gather, weights, bias, M, K):
        """The activation a x^2 + b x + c (a, b, c None: the square) followed by layer_conv_dense, with one relinearisation per output
        instead of one per input (include/cnhe.h, cnhe_layer_activation_conv_dense).  a, b, c as for layer_poly2; the outputs have scale
        scale(a) s^2 scale(w), which the bias must share."""
        g = None
        if gather is not None:
            g = np.ascontiguousarray(gather, dtype=np.int32)
            assert g.size == M * K
        out = (VECP * M)()
        h = lambda v: None if v is None else v.h
        check(self.L.cnhe_layer_activation_conv_dense(
            self.h, _vec_array(inputs), len(inputs), h(a), h(b), h(c), None if g is None else g.ctypes.data_as(C.POINTER(C.c_int32)),
            _vec_array(weights), None if bias is None else _vec_array(bias), M, K, out))
        return self._wrap_many(out, M)

    def _wrap_many(self, out, n, like=None):
        """Vec handles for the n outputs of one batched call: they share dim/scale/format/blocks, so the metadata is queried once.
        like: the inputs of a call whose outputs follow their own input's shape -- shared only when those inputs share theirs."""
        vecs = [Vec(self, out[i]) for i in range(n)]
        if like is not None and any(v.meta() != like[0].meta() for v in like[1:]):
            return vecs
        if n > 1:
            m = vecs[0].meta()
            for v in vecs[1:]:
                v._m = m
        return vecs

    def layer_square(self, inputs):
        n = len(inputs)
        out = (VECP * n)()
        check(self.L.cnhe_layer_square(self.h, _vec_array(inputs), n, out))
        return self._wrap_many(out, n, like=inputs)

    def layer_poly2(self, inputs, a, b=None, c=None):
        """a x^2 + b x + c of every input in layer_square's passes (include/cnhe.h, cnhe_layer_poly2): a, b, c are plain sparse vectors of
        dimension 1 at scales W, W s and W s^2 (b, c may be None); the outputs have scale W s^2."""
        n = len(inputs)
        out = (VECP * n)()
        h = lambda v: None if v is None else v.h
        check(self.L.cnhe_layer_poly2(self.h, _vec_array(inputs), n, h(a), h(b), h(c), out))
        return self._wrap_many(out, n, like=inputs)

    def layer_poly(self, inputs, coeffs):
        """P(x) = sum_j coeffs[j] x^j of every input, degree len(coeffs) - 1 = 3 or 4, in two levels of squares (include/cnhe.h,
        cnhe_layer_poly): coeffs[j] is a plain sparse vector of dimension 1 at scale W s^(degree - j), or None for 0 (the leading one is
        required); the outputs have scale W s^degree."""
        n = len(inputs)
        out = (VECP * n)()
        check(self.L.cnhe_layer_poly(self.h, _vec_array(inputs), n, _vec_array(list(coeffs)), len(coeffs) - 1, out))
        return self._wrap_many(out, n, like=inputs)

    # ---- raw device arrays (micro-benchmarks, kernel parity tests)
    def dev_alloc(self, words):
        p = C.c_uint64()
        check(self.L.cnhe_dev_alloc(self.h, int(words), C.byref(p)))
        return p.value

    def dev_free(self, ptr):
        check(self.L.cnhe_dev_free(self.h, int(ptr)))

    def dev_upload(self, ptr, data):
        a = _u64(data).ravel()
        check(self.L.cnhe_dev_upload(self.h, int(ptr), _p(a), a.size))

    def dev_download(self, ptr, words):
        a = np.zeros(int(words), np.uint64)
        check(self.L.cnhe_dev_download(self.h, _p(a), int(ptr), a.size))
        return a

    def dev_from(self, data):
        a = _u64(data).ravel()
        p = self.dev_alloc(a.size)
        self.dev_upload(p, a)
        return p

    def raw_ntt(self, src, dst, n_polys, mod_base, mod_count, inverse=False):
        check(self.L.cnhe_raw_ntt(self.h, int(src), int(dst), int(n_polys), int(mod_base), int(mod_count), int(inverse)))

    def raw_multiply(self, ch, a, b, n, out3):
        check(self.L.cnhe_raw_multiply(self.h, ch, int(a), int(b), int(n), int(out3)))

    def raw_relinearize(self, ch, in3, n, out2):
        check(self.L.cnhe_raw_relinearize(self.h, ch, int(in3), int(n), int(out2)))

    def raw_multiply_relin(self, ch, a, b, n, out2):
        check(self.L.cnhe_raw_multiply_relin(self.h, ch, int(a), int(b), int(n), int(out2)))

    def raw_apply_galois(self, ch, src, n, elt, out):
        check(self.L.cnhe_raw_apply_galois(self.h, ch, int(src), int(n), int(elt), int(out)))

    def raw_rotate_rows(self, ch, src, n, steps, out):
        check(self.L.cnhe_raw_rotate_rows(self.h, ch, int(src), int(n), int(steps), int(out)))

    def raw_behz_lift(self, src, n, out):
        check(self.L.cnhe_raw_behz_lift(self.h, int(src), int(n), int(out)))

    def raw_behz_floor(self, ch, d, n, out3):
        check(self.L.cnhe_raw_behz_floor(self.h, ch, int(d), int(n), int(out3)))

    def raw_import_products(self, words, n, dim=None, scale=1.0, slot=0):
        """n size-3 products (words [P][n][3][k][N]) as pending squares of one group in key slot `slot` (include/cnhe.h,
        cnhe_raw_import_products): a scalar-MAC layer over them takes the exact path, any other read relinearises them."""
        a = _u64(words).ravel()
        assert a.size == self.P * n * 3 * self.k * self.N
        out = (VECP * n)()
        check(self.L.cnhe_raw_import_products(self.h, _p(a), int(n), int(self.N if dim is None else dim), float(scale), int(slot), out))
        return self._wrap_many(out, n)

    def timer_start(self):
        check(self.L.cnhe_raw_event_timing(self.h, 1))

    def timer_stop_ms(self):
        check(self.L.cnhe_raw_event_timing(self.h, 0))
        ms = C.c_float()
        check(self.L.cnhe_raw_elapsed_ms(self.h, C.byref(ms)))
        return ms.value
