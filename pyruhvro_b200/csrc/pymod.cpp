// CPython extension `pyruhvro_b200._native`: the part of the reference's PyO3 layer that has to
// be native — walking a Python list[bytes] and releasing the GIL around the decode.
//
// Mirrors src/lib.rs of the reference:
//   extract_bytes_list  (:29-33)  elements must be `bytes`
//   py.detach(...)      (:64-69,82-87)  the GIL is released around the decode (packing keeps it: see pack_list)
//   to_py_err           (:25-27)  failures surface as ValueError(str)
// Packing into one contiguous buffer + offsets is what the reference itself does with
// BinaryArray::from_vec (ruhvro/src/deserialize.rs:90); here it lands in pinned host memory so
// the H2D copy runs at PCIe speed.
#define PY_SSIZE_T_CLEAN
#include <Python.h>

#include <algorithm>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <thread>
#include <stdexcept>
#include <vector>

#include "ruhvro_b200.h"

namespace {

// Packs a list[bytes] into one contiguous buffer + i64 offsets (what BinaryArray::from_vec builds at
// ruhvro/src/deserialize.rs:90).  The GIL is HELD for the whole function: the elements are only borrowed, and
// nothing can mutate the list or free an element while no other Python thread can run — so the walk is one
// read of each object header (type, size, payload pointer) with no INCREF/DECREF passes, which were two thirds of
// its cost.  The payload gather fans out over plain C++ threads (they touch no Python state).
// `alloc(bytes)` returns the destination memory (pinned for the decode path).  Returns false with a Python
// exception set.
struct JoinAll {  // joins whatever was started, also when starting a later thread throws
    std::vector<std::thread>& th;
    ~JoinAll() { for (auto& t : th) if (t.joinable()) t.join(); }
};

struct Packed {
    char* data = nullptr;
    int64_t* offsets = nullptr;
    int64_t total = 0;
    Py_ssize_t n = 0;
};

template <class Alloc>
bool pack_list(PyObject* list, Alloc alloc, Packed* out) {
    const Py_ssize_t n = PyList_GET_SIZE(list);
    out->n = n;
    out->offsets = static_cast<int64_t*>(alloc((static_cast<size_t>(n) + 1) * 8));
    if (!out->offsets) {
        PyErr_SetString(PyExc_ValueError, "pinned host allocation failed (is a CUDA device present?)");
        return false;
    }
    std::unique_ptr<const char*[]> ptrs(new const char*[static_cast<size_t>(n) + 1]);  // uninitialised on purpose
    int64_t* offsets = out->offsets;
    offsets[0] = 0;
    const unsigned hw = std::min(16u, std::max(1u, std::thread::hardware_concurrency()));
    // One read of every element's header: type check, payload pointer, size (left in offsets[i + 1]).  Long lists are
    // walked by several threads — the calling thread holds the GIL throughout, so nothing they read can change.
    auto walk = [list, offsets, p = ptrs.get()](Py_ssize_t a, Py_ssize_t b) -> Py_ssize_t {  // -> first element that is neither bytes nor bytearray, or b
        for (Py_ssize_t i = a; i < b; ++i) {
            PyObject* item = PyList_GET_ITEM(list, i);
            if (PyBytes_Check(item)) {
                p[static_cast<size_t>(i)] = PyBytes_AS_STRING(item);
                offsets[i + 1] = static_cast<int64_t>(PyBytes_GET_SIZE(item));
            } else if (PyByteArray_Check(item)) {
                // PyBackedBytes (what the reference extracts, src/lib.rs:29-33) takes `bytes` or `bytearray`.  The payload is
                // copied below while this call still holds the GIL, so the array cannot change size meanwhile.
                p[static_cast<size_t>(i)] = PyByteArray_AS_STRING(item);
                offsets[i + 1] = static_cast<int64_t>(PyByteArray_GET_SIZE(item));
            } else {
                return i;
            }
        }
        return b;
    };
    Py_ssize_t bad = n;
    if (n < (Py_ssize_t(1) << 16) || hw <= 1) {
        bad = walk(0, n);
    } else {
        std::vector<Py_ssize_t> stop(hw, 0);
        std::vector<std::thread> th;
        JoinAll join_all{th};
        for (unsigned w = 0; w < hw; ++w) {
            const Py_ssize_t a = n / Py_ssize_t(hw) * Py_ssize_t(w), b = (w + 1 == hw) ? n : n / Py_ssize_t(hw) * Py_ssize_t(w + 1);
            th.emplace_back([&stop, &walk, w, a, b] { const Py_ssize_t r = walk(a, b); stop[w] = r == b ? -1 : r; });
        }
        for (auto& t : th) t.join();
        for (unsigned w = hw; w-- > 0;) if (stop[w] >= 0) bad = stop[w];   // the lowest failing index wins
    }
    if (bad < n) {
        PyErr_Format(PyExc_TypeError, "argument 'list': element %zd is '%s', expected 'bytes' or 'bytearray'", bad, Py_TYPE(PyList_GET_ITEM(list, bad))->tp_name);
        return false;
    }
    for (Py_ssize_t i = 0; i < n; ++i) offsets[i + 1] += offsets[i];
    const int64_t total = offsets[n];
    out->total = total;
    out->data = static_cast<char*>(alloc(static_cast<size_t>(total) + 64));
    if (!out->data) {
        PyErr_SetString(PyExc_ValueError, "pinned host allocation failed (is a CUDA device present?)");
        return false;
    }
    const unsigned workers = total > (int64_t(8) << 20) ? hw : 1u;
    char* dst = out->data;
    const char* const* src = ptrs.get();
    auto copy_range = [dst, src, offsets](Py_ssize_t a, Py_ssize_t b) {
        for (Py_ssize_t i = a; i < b; ++i) std::memcpy(dst + offsets[i], src[i], static_cast<size_t>(offsets[i + 1] - offsets[i]));
    };
    if (workers <= 1) {
        copy_range(0, n);
    } else {
        // split by BYTES, not by element count, so skewed inputs still balance
        std::vector<std::thread> th;
        JoinAll join_all{th};
        Py_ssize_t a = 0;
        for (unsigned w = 0; w < workers; ++w) {
            const int64_t want = total / int64_t(workers) * int64_t(w + 1);
            const Py_ssize_t b = (w + 1 == workers) ? n : Py_ssize_t(std::upper_bound(offsets, offsets + n + 1, want) - offsets - 1);
            const Py_ssize_t bb = std::max(a, std::min(b, n));
            th.emplace_back(copy_range, a, bb);
            a = bb;
        }
        for (auto& t : th) t.join();
    }
    return true;
}

struct PinnedPair {  // the two slabs of one call
    void* a = nullptr;
    void* b = nullptr;
    ~PinnedPair() { rv_host_free(a); rv_host_free(b); }
};

// The pinned gather of `list`, then decode(data, offsets, n, &result) without the GIL (py.detach, src/lib.rs:64-69,82-87).
// Returns the result handle (int), or nullptr with the Python error set.
template <class Decode>
PyObject* decode_gathered(PyObject* list, Decode&& decode) {
    PinnedPair slabs;
    Packed pk;
    bool first = true;
    auto alloc = [&](size_t bytes) -> void* {
        void* p = rv_host_alloc(bytes);
        (first ? slabs.a : slabs.b) = p;
        first = false;
        return p;
    };
    try {
        if (!pack_list(list, alloc, &pk)) return nullptr;
    } catch (const std::exception& e) {  // bad_alloc, std::system_error from std::thread: a Python error, not an abort
        PyErr_SetString(PyExc_MemoryError, e.what());
        return nullptr;
    }
    rv_result* result = nullptr;
    rv_status st = RV_OK;
    Py_BEGIN_ALLOW_THREADS;
    st = decode(reinterpret_cast<const uint8_t*>(pk.data), pk.offsets, pk.n, &result);
    Py_END_ALLOW_THREADS;
    if (st != RV_OK) {
        PyErr_SetString(PyExc_ValueError, rv_last_error());
        return nullptr;
    }
    return PyLong_FromUnsignedLongLong(static_cast<unsigned long long>(reinterpret_cast<uintptr_t>(result)));
}

// decode_list(schema_handle: int, records: list[bytes], num_chunks: int) -> result handle (int)
PyObject* decode_list(PyObject*, PyObject* args) {
    unsigned long long schema_addr = 0;
    PyObject* list = nullptr;
    long long num_chunks = 1, header_bytes = 0, check_magic = 0, schema_id = -1;
    if (!PyArg_ParseTuple(args, "KO!L|LLL", &schema_addr, &PyList_Type, &list, &num_chunks, &header_bytes, &check_magic, &schema_id)) return nullptr;
    const rv_schema* schema = reinterpret_cast<const rv_schema*>(static_cast<uintptr_t>(schema_addr));
    const rv_framing framing = {int32_t(header_bytes), int32_t(check_magic), int64_t(schema_id)};
    return decode_gathered(list, [&](const uint8_t* data, const int64_t* offsets, int64_t n, rv_result** out) {
        return rv_decode_host_framed(schema, data, offsets, n, num_chunks, header_bytes > 0 ? &framing : nullptr, out);
    });
}

// decode_list_versions(versions_handle: int, records: list[bytes], num_chunks: int) -> result handle (int): Confluent or
// single-object messages of several writer schemas (rv_decode_host_versions), through the same pinned gather as decode_list
PyObject* decode_list_versions(PyObject*, PyObject* args) {
    unsigned long long addr = 0;
    PyObject* list = nullptr;
    long long num_chunks = 1;
    if (!PyArg_ParseTuple(args, "KO!L", &addr, &PyList_Type, &list, &num_chunks)) return nullptr;
    const rv_versions* v = reinterpret_cast<const rv_versions*>(static_cast<uintptr_t>(addr));
    return decode_gathered(list, [&](const uint8_t* data, const int64_t* offsets, int64_t n, rv_result** out) {
        return rv_decode_host_versions(v, data, offsets, n, num_chunks, out);
    });
}

// decode_list_single_object(schema_handle: int, records: list[bytes], num_chunks: int) -> result handle (int): Avro
// single-object messages of one writer schema (rv_decode_host_single_object)
PyObject* decode_list_single_object(PyObject*, PyObject* args) {
    unsigned long long schema_addr = 0;
    PyObject* list = nullptr;
    long long num_chunks = 1;
    if (!PyArg_ParseTuple(args, "KO!L", &schema_addr, &PyList_Type, &list, &num_chunks)) return nullptr;
    const rv_schema* schema = reinterpret_cast<const rv_schema*>(static_cast<uintptr_t>(schema_addr));
    return decode_gathered(list, [&](const uint8_t* data, const int64_t* offsets, int64_t n, rv_result** out) {
        return rv_decode_host_single_object(schema, data, offsets, n, num_chunks, out);
    });
}

// pack(records: list[bytes]) -> (data: bytes, offsets: bytes of int64[n+1]).  The packing step alone, into ordinary
// memory: lets the CPU test-suite check the list walk / gather without a GPU.
PyObject* pack(PyObject*, PyObject* args) {
    PyObject* list = nullptr;
    if (!PyArg_ParseTuple(args, "O!", &PyList_Type, &list)) return nullptr;
    std::vector<void*> blocks;
    auto alloc = [&](size_t bytes) -> void* { void* p = std::malloc(bytes ? bytes : 1); blocks.push_back(p); return p; };
    Packed pk;
    PyObject* out = nullptr;
    bool ok = false;
    try {
        ok = pack_list(list, alloc, &pk);
    } catch (const std::exception& e) {
        PyErr_SetString(PyExc_MemoryError, e.what());
    }
    if (ok)
        out = Py_BuildValue("(y#y#)", pk.data, static_cast<Py_ssize_t>(pk.total), reinterpret_cast<const char*>(pk.offsets),
                            static_cast<Py_ssize_t>((static_cast<size_t>(pk.n) + 1) * 8));
    for (void* p : blocks) std::free(p);
    return out;
}

PyMethodDef methods[] = {
    {"decode_list", decode_list, METH_VARARGS, "decode_list(schema_handle, records: list[bytes], num_chunks[, header_bytes, check_magic, schema_id]) -> result handle"},
    {"decode_list_versions", decode_list_versions, METH_VARARGS, "decode_list_versions(versions_handle, records: list[bytes], num_chunks) -> result handle"},
    {"decode_list_single_object", decode_list_single_object, METH_VARARGS, "decode_list_single_object(schema_handle, records: list[bytes], num_chunks) -> result handle"},
    {"pack", pack, METH_VARARGS, "pack(records: list[bytes]) -> (data, offsets): the packing step alone (test hook)"},
    {nullptr, nullptr, 0, nullptr},
};

PyModuleDef moddef = {PyModuleDef_HEAD_INIT, "_native", "list[bytes] packing + GIL release for pyruhvro_b200", -1, methods, nullptr, nullptr, nullptr, nullptr};

}  // namespace

PyMODINIT_FUNC PyInit__native(void) { return PyModule_Create(&moddef); }
