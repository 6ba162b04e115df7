/*
 * ruhvro_b200.h — C ABI of the H100-native Avro -> Arrow direct decoder.
 *
 * This is the drop-in boundary for the reference's direct-decode hot path: every entry
 * point names the reference interface it replaces (file:line in Tyler-Sch/pyruhvro @ de4683de).
 * A Rust `extern "C"` shim inside `ruhvro::deserialize` (or the ctypes/CPython binding in
 * pyruhvro_b200/) binds these 1:1 — see INTEGRATION.md.
 *
 * Conventions
 *   - Plain pointers and sizes only; no C++/torch types.  All functions are thread-safe and
 *     never throw or abort across the boundary.
 *   - Status 0 = success; non-zero = the error category below.  rv_last_error() returns the
 *     calling thread's last message (the analogue of the reference's anyhow::Error string,
 *     surfaced to Python as ValueError at src/lib.rs:25-27).
 *   - Inputs are borrowed for the duration of the call.  Outputs are owned by the library and
 *     released through rv_result_free() and the Arrow C Data Interface release callbacks.
 *   - There is NO CPU fallback: schemas outside the direct-decode subset
 *     (fast_decode.rs:38-61) are an error here, where the reference would drop to its
 *     Value-tree path (deserialize.rs:26-29).  A missing CUDA device is an error.
 */
#ifndef RUHVRO_B200_H
#define RUHVRO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

struct ArrowSchema;      /* Arrow C Data Interface (pyruhvro_b200/csrc/arrow_c.h) */
struct ArrowArray;
struct ArrowDeviceArray; /* Arrow C Device Data Interface */

typedef struct rv_schema rv_schema; /* parsed Avro schema + decode plan; immutable, ref-counted */
typedef struct rv_result rv_result; /* the k RecordBatches of one decode call */
typedef struct rv_encoded rv_encoded; /* the k Binary arrays (or the container file) of one encode call */

typedef enum rv_status {
    RV_OK = 0,
    /* data errors: categories of the reference's bail!/anyhow! sites in fast_decode.rs */
    RV_ERR_EOF = 1,          /* :849,874,884,910 "unexpected end of buffer" */
    RV_ERR_VARINT = 2,       /* :866 "zigzag varint too long" */
    RV_ERR_BOOL = 3,         /* :898 "invalid boolean byte" */
    RV_ERR_NEG_LEN = 4,      /* :906 "negative string length" */
    RV_ERR_BRANCH = 5,       /* :591,646 union branch index invalid / out of range */
    RV_ERR_ENUM = 6,         /* :575 "enum index out of range" */
    RV_ERR_SCHEMA = 7,       /* schema does not parse / outside the supported subset / over a documented limit */
    RV_ERR_OVERFLOW = 8,     /* a column of one batch exceeds Arrow's i32 offsets (arrow-rs panics here) */
    RV_ERR_INVALID = 9,      /* bad argument */
    RV_ERR_CUDA = 10,        /* CUDA runtime failure (includes "no device") */
    RV_ERR_VALUE = 11,       /* wider subset: uuid text that is not a UUID, decimal wider than 128 bits */
    RV_ERR_FRAME = 12        /* framed input: message shorter than its header, wrong magic byte, unexpected schema id or fingerprint */
} rv_status;

/* ---- schema --------------------------------------------------------------------------- */

/* Replaces ruhvro::deserialize::parse_schema (ruhvro/src/deserialize.rs:18-20).  Parsing an
 * unsupported-but-valid schema succeeds; use rv_schema_is_supported() for the gate.  A document
 * apache-avro's Schema::parse_str turns away is RV_ERR_SCHEMA here too: malformed JSON, missing
 * attributes, type / field names and enum symbols outside [A-Za-z_][A-Za-z0-9_]*, repeated field
 * names or enum symbols, duplicate unnamed kinds or a nested union in a union.  (Not checked:
 * record field defaults against the field's type.) */
rv_status rv_schema_parse(const char* json, size_t len, rv_schema** out);
rv_schema* rv_schema_retain(rv_schema* s);  /* Arc::clone (deserialize.rs:96) */
void rv_schema_release(rv_schema* s);

/* Replaces fast_decode::is_supported (ruhvro/src/fast_decode.rs:38-61): 1 = decodable here. */
int rv_schema_is_supported(const rv_schema* s);

/* Replaces schema_translate::to_arrow_schema (ruhvro/src/schema_translate.rs:19-37): exports
 * the Arrow schema ("+s" struct of the top-level fields) of the batches decode returns. */
rv_status rv_schema_export_arrow(const rv_schema* s, struct ArrowSchema* out);

/* Column projection: a new, independent handle (release it with rv_schema_release) whose batches hold only the
 * top-level fields named in columns[0 .. n_columns), in that order.  Rows and chunking are unchanged, and every column
 * is buffer for buffer the column of the full decode.  The other fields are still read and validated with the same
 * checks as in a full decode, so a projected decode fails on the same record with the same status; the one exception
 * is RV_ERR_OVERFLOW, which only a column that is produced can raise.  A selected record / list / map / union column
 * comes out whole; nested paths ("address.city") are not supported.
 * The handle works with every decode entry point (host, device, framed, rv_gather_*), rv_schema_export_arrow (the
 * selected fields, same metadata), rv_schema_walker_source and rv_schema_precompile; rv_encode_host refuses it
 * (RV_ERR_INVALID).  Projecting a projected handle selects among its columns.
 * RV_ERR_INVALID: an empty list, a repeated name or a name that is not a top-level field (the message lists the
 * fields).  RV_ERR_SCHEMA: `s` is not decodable. */
rv_status rv_schema_project(const rv_schema* s, const char* const* columns, int64_t n_columns, rv_schema** out);

/* Schema resolution (the Avro specification's "Schema Resolution", restricted as DESIGN.md §7 lists): a new, independent
 * handle that walks datums as the WRITER's schema lays them out and returns batches in the READER's Arrow form.  A resolved
 * decode of a datum gives the same batch, buffer for buffer, as decoding it with the writer's schema, converting the value
 * (promotions int -> long / float / double, long -> float / double with one round-to-nearest-even step, float -> double,
 * string <-> bytes; enum symbols by name; record fields by name or reader alias, in the reader's order; reader-only fields
 * from their "default"; a writer non-union read as a reader ["null", T] is never null), encoding it with the reader's
 * schema and decoding that.  Writer-only fields are read and validated as in a full decode and produce nothing.
 * A resolved decode fails on the same record with the same status as a decode with the writer's schema, except that
 * RV_ERR_OVERFLOW only comes from produced columns, and a writer enum symbol the reader has neither a symbol nor a
 * default for is RV_ERR_ENUM "(record N)".
 * The handle works with every decode entry point, rv_gather_*, rv_schema_export_arrow (exactly the reader's own
 * schema), rv_schema_walker_source / kernel_source / max_tile / precompile and rv_schema_project (the reader's top-level
 * fields); rv_encode_host refuses it (RV_ERR_INVALID).
 * A reader-only field of a union type whose first branch is null may default to null whatever else the union holds
 * (a null record, list, fixed, decimal or uuid); other defaults must be leaf values.
 * RV_ERR_SCHEMA, naming the reader field's path ("address.country"): a pair outside the rules, a reader-only field
 * without a default or with one that does not match its type or is a record / list / map / fixed / decimal / uuid
 * value, unions with branches added, removed or reordered, a
 * writer union read as a non-union, promotions between logical types.  RV_ERR_INVALID: a projected or resolved handle
 * passed as writer or reader. */
rv_status rv_schema_resolve(const rv_schema* writer, const rv_schema* reader, rv_schema** out);

/* A permissive handle: decodes that do not fail on a damaged record.  Let R be the output schema of `s` (plain,
 * projected or resolved) and R' be R with every top-level field whose type is not a union, null or a map made optional
 * (T -> ["null", T]; a reader-only field with a non-null default -> [T, "null"], the same Arrow column; a nullable map
 * has no Arrow form here).  Every
 * rv_decode_{host,device}[_framed|_single_object] entry point takes the handle.  Each record whose strict decode alone
 * fails with RV_ERR_EOF, _VARINT, _BOOL, _NEG_LEN, _BRANCH, _ENUM (an unmapped enum symbol included), _VALUE or _FRAME
 * becomes a bad row: null in every top-level column (a map column: an empty map; an N-variant union column: type id 0
 * and absent children), listed by rv_result_bad.  Other rows hold the strict decode's values; the k batches keep the strict call's row counts, so
 * rows stay aligned with the input messages.  RV_ERR_OVERFLOW, RV_ERR_SCHEMA, RV_ERR_INVALID and RV_ERR_CUDA still
 * fail the call.  The batches are, buffer for buffer, the plain decode with R' of the input in which every good record
 * is re-encoded with R' and every bad one is the datum with branch null in each optional top-level field.
 * rv_schema_export_arrow gives R'; the canonical form and fingerprint stay the writer's.  rv_schema_project of a
 * permissive handle stays permissive.  RV_ERR_INVALID: `s` is already permissive.  rv_versions_create*, rv_encode_*
 * and rv_encode_ocf_host refuse a permissive handle (RV_ERR_INVALID). */
rv_status rv_schema_permissive(const rv_schema* s, rv_schema** out);

/* The Avro specification's Parsing Canonical Form of the schema and its CRC-64-AVRO fingerprint (the 64-bit Rabin
 * fingerprint, EMPTY = 0xc15d213aa4d7a795), the key single-object encoding names a writer schema by.  The form keeps
 * primitives as bare names, named types by fullname (in full at their first occurrence, by fullname after that), only
 * name / type / fields / symbols / items / values / size in that order, and drops namespaces, logical types, docs,
 * aliases, defaults and whitespace.  Schemas that differ only in what is dropped share a fingerprint.
 * For a projected or resolved handle both describe the writer's full schema: the schema the messages were written with.
 * rv_schema_canonical_form returns the form's length and copies at most cap-1 bytes + NUL into buf (buf may be NULL).
 * A schema with a construct the parser keeps as unsupported (duration, local-timestamp-*, timestamp-nanos, a recursive
 * type, ...) has no form here: -1 / RV_ERR_SCHEMA. */
int64_t rv_schema_canonical_form(const rv_schema* s, char* buf, size_t cap);
rv_status rv_schema_fingerprint(const rv_schema* s, uint64_t* out);

/* ---- decode ---------------------------------------------------------------------------- */

/* Replaces ruhvro::deserialize::per_datum_deserialize_threaded (ruhvro/src/deserialize.rs:76-121)
 * and, with num_chunks = 1, per_datum_deserialize (:25-30).
 *
 * `data`/`offsets` are the packed form the reference itself builds with BinaryArray::from_vec
 * (:90): record i is data[offsets[i] .. offsets[i+1]), offsets has n+1 entries (i64, so inputs
 * beyond 2 GiB are addressable).  num_chunks is clamped like clamp_chunks (:53-55) and rows are
 * partitioned like build_slices (:57-68): chunk = n / k, the last chunk takes the remainder;
 * one RecordBatch per chunk, in order.  n = 0 yields one empty batch.
 *
 * Host variant: `data`/`offsets` are host memory.  Page-locked memory (rv_host_alloc, cudaHostAlloc,
 * cudaHostRegister) is copied from directly; ordinary pageable memory (a Rust Vec, a numpy array) is
 * recognised and uploaded through the library's pinned staging pieces, overlapped with the transfer.
 * The batches' buffers land in library-owned pinned host memory. */
rv_status rv_decode_host(const rv_schema* s, const uint8_t* data, const int64_t* offsets, int64_t n,
                         int64_t num_chunks, rv_result** out);

/* Device variant (the benchmark / pipeline path): `d_data`/`d_offsets` are device pointers on the
 * current CUDA device, `d_data` 16-byte aligned and readable for at least 16 bytes past
 * d_data[d_offsets[n]] (tiles are staged in 16-byte vectors); work is enqueued on `cuda_stream` (a
 * cudaStream_t; NULL = default stream) and the call returns after the kernels completed.  The
 * batches stay in HBM until rv_result_to_host(); their buffers are sized from what earlier calls on
 * the same schema handle needed, so they may carry a few per cent of slack between them. */
rv_status rv_decode_device(const rv_schema* s, const uint8_t* d_data, const int64_t* d_offsets, int64_t n,
                           int64_t num_chunks, void* cuda_stream, rv_result** out);

/* Framed inputs (SURVEY.md 8(f) rank 4) — the step before the path in Kafka pipelines.  The reference takes bare datums
 * only (README.md:93-94: callers strip the Confluent header themselves, one Python slice per message); here the strip is
 * offset arithmetic inside the decode kernel: record i is still data[offsets[i] .. offsets[i+1]), but its datum starts
 * `header_bytes` later.  check_magic != 0 validates the Confluent wire format's header (byte 0 = 0x00; with
 * schema_id >= 0 also the big-endian u32 schema id in bytes 1..4): a mismatch is RV_ERR_FRAME with the record index. */
typedef struct rv_framing {
    int32_t header_bytes;  /* bytes to skip at the start of every message (Confluent: 5) */
    int32_t check_magic;   /* 0: skip only; 1: check the Confluent magic byte (and the id when schema_id >= 0) */
    int64_t schema_id;     /* -1: any */
} rv_framing;
rv_status rv_decode_host_framed(const rv_schema* s, const uint8_t* data, const int64_t* offsets, int64_t n,
                                int64_t num_chunks, const rv_framing* framing, rv_result** out);
rv_status rv_decode_device_framed(const rv_schema* s, const uint8_t* d_data, const int64_t* d_offsets, int64_t n,
                                  int64_t num_chunks, const rv_framing* framing, void* cuda_stream, rv_result** out);

/* Avro single-object encoding: every message is C3 01, the little-endian CRC-64-AVRO fingerprint of the writer's schema
 * (rv_schema_fingerprint of `s`: the writer's, also for a projected or resolved handle), then the datum.  The header is
 * checked and skipped inside the decode kernel.  A message shorter than 10 bytes, not starting with C3 01 or naming
 * another fingerprint is RV_ERR_FRAME with its record index; the lowest failing record wins as on every path.
 * RV_ERR_SCHEMA: a schema without a canonical form.  Otherwise rv_decode_host / rv_decode_device. */
rv_status rv_decode_host_single_object(const rv_schema* s, const uint8_t* data, const int64_t* offsets, int64_t n,
                                       int64_t num_chunks, rv_result** out);
rv_status rv_decode_device_single_object(const rv_schema* s, const uint8_t* d_data, const int64_t* d_offsets, int64_t n,
                                         int64_t num_chunks, void* cuda_stream, rv_result** out);

/* An Avro Object Container File (magic, header with avro.schema / avro.codec, blocks of datums between sync markers;
 * uncompressed blocks only) -> `num_chunks` batches in pinned host memory.  The schema comes from the file: a new handle is
 * returned in *schema_out (release it with rv_schema_release).  Datums inside a block carry no lengths: the host walks
 * the block headers, a kernel with one lane per block walks the records to find their offsets, then the decode kernel
 * runs as on any packed input.  A malformed container is RV_ERR_FRAME, and so is a block that claims more records than
 * it has bytes (checked on the host, before any CUDA call): every datum takes at least one byte, so a container of a
 * schema whose datums are always empty (records of null fields only) holds no records.  A record that fails to decode
 * reports the error of the lowest failing record, "(record N)"; a block whose records end before its byte size is
 * RV_ERR_FRAME at the block's last record. */
rv_status rv_decode_ocf_host(const uint8_t* file, int64_t len, int64_t num_chunks, rv_schema** schema_out, rv_result** out);

/* rv_decode_ocf_host with a column projection (rv_schema_project) of the file's schema: *schema_out is the projected
 * handle.  Record offsets are still found by walking every byte of every record. */
rv_status rv_decode_ocf_host_projected(const uint8_t* file, int64_t len, int64_t num_chunks, const char* const* columns,
                                       int64_t n_columns, rv_schema** schema_out, rv_result** out);
/* The file's records read with `reader` (rv_schema_resolve: the file's schema is the writer's), optionally projected to
 * the reader's top-level fields columns[0 .. n_columns) (columns may be NULL with n_columns 0).  The record offsets are
 * still found by walking the writer's schema.  *schema_out is the resolved (and projected) handle. */
rv_status rv_decode_ocf_host_resolved(const uint8_t* file, int64_t len, int64_t num_chunks, const rv_schema* reader,
                                      const char* const* columns, int64_t n_columns, rv_schema** schema_out, rv_result** out);

/* ---- several writer schemas: Confluent messages of a topic written with different schema versions ------------------
 * A registry: the reader's schema and, for each registered schema id, the writer's schema it names.  Immutable and
 * thread-safe once created; it keeps one resolved handle (rv_schema_resolve, projected to `columns` when given) per
 * writer, so each writer's capacity history and compiled walker persist across calls, and a walker is compiled only when
 * its id first appears in a call.
 * columns: the reader's top-level fields the batches hold (rv_schema_project; NULL with n_columns 0: all of them).
 * At most 256 writers.  Fails before any CUDA call:
 *   RV_ERR_INVALID: no writers, more than 256, an id outside [0, 2^32 - 1] or registered twice, a projected or resolved
 *                   handle as reader or writer, an unknown column;
 *   RV_ERR_SCHEMA:  a writer that does not resolve to the reader ("schema id X: " then rv_schema_resolve's message). */
typedef struct rv_versions rv_versions;
rv_status rv_versions_create(const rv_schema* reader, const int64_t* schema_ids, const rv_schema* const* writers,
                             int64_t n_writers, const char* const* columns, int64_t n_columns, rv_versions** out);
void rv_versions_release(rv_versions* v);
/* A registry of single-object writers, keyed by the fingerprints of writers[0 .. n_writers) (rv_schema_fingerprint).
 * Everything else is rv_versions_create's.  Fails before any CUDA call, RV_ERR_INVALID: two writers with the same
 * fingerprint (schemas that differ only in what the canonical form drops, which the wire cannot tell apart), no writers
 * or more than 256, a projected or resolved handle, an unknown column.  RV_ERR_SCHEMA: a writer without a canonical form,
 * a writer that does not resolve to the reader. */
rv_status rv_versions_create_single_object(const rv_schema* reader, const rv_schema* const* writers, int64_t n_writers,
                                           const char* const* columns, int64_t n_columns, rv_versions** out);
/* A permissive registry made from `v`: same keys, writers and columns; its batches are R' (rv_schema_permissive of the
 * reader, projected to the columns), and rv_decode_*_versions with it turns a bad message into a null row and reports
 * it (rv_result_num_bad / rv_result_bad / rv_result_bad_message) instead of failing the call.  A message is bad when
 * the strict decode of it alone, with `v`, fails with a framing error (short, wrong magic byte, or a schema id or
 * fingerprint that is not registered: RV_ERR_FRAME, whose message names the id or fingerprint) or a record error of its
 * writer's resolved decode (RV_ERR_EOF, _VARINT, _BOOL, _NEG_LEN, _BRANCH, _ENUM including an unmapped symbol, _VALUE).
 * Its row is what a permissive decode writes for a bad record: null in every top-level column, an empty map in a map
 * column, type id 0 with absent children in an N-variant union column.  The report is in message order; each message is
 * the strict one without "(record N)".  RV_ERR_OVERFLOW, RV_ERR_SCHEMA, RV_ERR_INVALID and RV_ERR_CUDA still fail the
 * call.  `v` is unchanged and independent of the result.  RV_ERR_INVALID: `v` is already permissive. */
rv_status rv_versions_permissive(const rv_versions* v, rv_versions** out);

/* n Confluent messages (0x00, the big-endian u32 schema id, the datum) -- or, for a single-object registry, n
 * single-object messages (C3 01, the writer's fingerprint, the datum) -- -> num_chunks batches in the reader's Arrow form
 * (rv_schema_export_arrow of the reader, projected to the registry's columns), rows in message order.  Chunking is
 * rv_decode_host's; row j of batch i is message i * floor(n / k) + j decoded with the writer schema its id names and
 * resolved to the reader.  Batch i equals, buffer for buffer, the reader's decode of those messages each resolved and
 * re-encoded with the reader's schema.
 * Errors: the lowest failing message wins across every category, "(record N)" with N its index in the call.
 *   RV_ERR_FRAME: a message shorter than 5 bytes or with a wrong magic byte, or whose id is not registered ("schema id
 *                 X is not registered"); single-object: shorter than 10 bytes, not C3 01, or a fingerprint that is not
 *                 registered ("schema fingerprint 0x... is not registered");
 *   otherwise the status the message's writer's resolved decode gives for it (RV_ERR_ENUM for an unmapped symbol);
 *   RV_ERR_OVERFLOW: a column of an output batch exceeds Arrow's i32 offsets.
 * The messages are partitioned on the GPU into one group per (batch, writer), each group is decoded with its writer's
 * resolved handle, and a take interleaves the groups' rows back into message order.  When every message carries the
 * same id the input is decoded directly with that writer's handle.  Inputs, alignment and result ownership are those of
 * rv_decode_host / rv_decode_device. */
rv_status rv_decode_host_versions(const rv_versions* v, const uint8_t* data, const int64_t* offsets, int64_t n,
                                  int64_t num_chunks, rv_result** out);
rv_status rv_decode_device_versions(const rv_versions* v, const uint8_t* d_data, const int64_t* d_offsets, int64_t n,
                                    int64_t num_chunks, void* cuda_stream, rv_result** out);
/* CUDA-event timings of the calling thread's last rv_decode_*_versions call, in milliseconds: [0] partition, [1] the
 * groups' decodes (the whole decode on the single-id path), [2] take (0 on the single-id path), [3] all of it on the
 * device.  Returns how many entries were written. */
int rv_last_versions_timings(float* out_ms, int cap);

/* Copies a device-resident result's buffers to pinned host memory (no-op if already there). */
rv_status rv_result_to_host(rv_result* r);

int64_t rv_result_num_batches(const rv_result* r);
int64_t rv_result_num_rows(const rv_result* r, int64_t batch);
/* Exact bytes of every Arrow buffer that is exported (the B_out of the roofline bookkeeping). */
int64_t rv_result_arrow_bytes(const rv_result* r);

/* Permissive decodes (rv_schema_permissive): the bad records of the call, in record order.  rv_result_bad copies at most
 * `cap` of them (record index in the call, rv_status of the record's strict decode) and returns how many there are
 * (-1: a null argument with cap > 0).  rv_result_bad_message gives entry i's message: the strict call's message
 * without " (record N)" (NULL: no such entry).  A strict decode has none. */
int64_t rv_result_num_bad(const rv_result* r);
int64_t rv_result_bad(const rv_result* r, int64_t* records, int32_t* status, int64_t cap);
const char* rv_result_bad_message(const rv_result* r, int64_t i);

/* Bytes of the result's buffer arena (what rv_result_to_host copies over PCIe; includes 64-byte
 * padding and validity bitmaps that end up not being exported). */
int64_t rv_result_buffer_bytes(const rv_result* r);

/* Exports batch i as a struct array + (optionally, may be NULL) its schema through the Arrow C
 * Data Interface — what PyArrowType<RecordBatch> does at src/lib.rs:70,88.  Requires host buffers.
 * The exported array keeps the result's memory alive until its release callback runs. */
rv_status rv_result_export(rv_result* r, int64_t batch, struct ArrowArray* out_array, struct ArrowSchema* out_schema);
/* Same, for a device-resident result (device_type = ARROW_DEVICE_CUDA, buffers are device pointers). */
rv_status rv_result_export_device(rv_result* r, int64_t batch, struct ArrowDeviceArray* out_array, struct ArrowSchema* out_schema);

void rv_result_free(rv_result* r);

/* ---- encode (Arrow -> Avro) ----------------------------------------------------------------------------
 * Replaces ruhvro::serialize::serialize_record_batch (ruhvro/src/serialize.rs:38-67) + fast_encode::serialize_chunk
 * (ruhvro/src/fast_encode.rs:27-53) on the GPU.  `batch` / `batch_schema` are the RecordBatch as an Arrow C Data
 * struct array + schema (host buffers; slices/offsets allowed); OWNERSHIP MOVES to the callee, which releases
 * both.  Arrow columns are matched to Avro fields by NAME (fast_encode.rs:157-181); a missing column, a type the
 * reference's downcast would reject, an enum text outside the symbols or a union type id out of range are errors.
 * Rows are sliced into num_chunks chunks like slice_struct (:19-30); chunk i is exported as a Binary array
 * (i32 offsets + datum bytes), the GenericBinaryArray<i32> of the reference. */
/* A projected handle (rv_schema_project) is RV_ERR_INVALID. */
rv_status rv_encode_host(const rv_schema* s, struct ArrowArray* batch, struct ArrowSchema* batch_schema, int64_t num_chunks, rv_encoded** out);
int64_t rv_encoded_num_chunks(const rv_encoded* r);
rv_status rv_encoded_export(rv_encoded* r, int64_t chunk, struct ArrowArray* out_array, struct ArrowSchema* out_schema);
void rv_encoded_free(rv_encoded* r);
/* CUDA-event timings of the calling thread's last encode, in milliseconds: [0] size kernel, [1] scan, [2] write kernel
 * (with the container framing kernel), [3] upload of the Arrow buffers, [4] download of the datums.  Summed over row
 * groups.  Returns how many entries were written. */
int rv_last_encode_timings(float* out_ms, int cap);

/* Framed outputs, the write-side mirror of the framed inputs above (extensions: the reference has no such calls).  Both
 * follow rv_encode_host in everything not stated here: ownership of batch / batch_schema moves to the callee, columns
 * are matched by name, slices are honoured, errors are the same (the lowest failing row wins), and a projected or
 * resolved handle is RV_ERR_INVALID.
 *
 * Confluent wire format: every datum is preceded by 0x00 and the big-endian u32 schema_id.  Chunking is rv_encode_host's;
 * chunk i is exported by rv_encoded_export as a Binary array whose element j is the 5-byte header followed by the datum,
 * and the i32 overflow check of a chunk counts the headers.  schema_id outside [0, 2^32 - 1] is RV_ERR_INVALID. */
rv_status rv_encode_host_confluent(const rv_schema* s, struct ArrowArray* batch, struct ArrowSchema* batch_schema,
                                   int64_t num_chunks, int64_t schema_id, rv_encoded** out);

/* Avro single-object encoding: every datum is preceded by C3 01 and the little-endian CRC-64-AVRO fingerprint of `s`
 * (rv_schema_fingerprint), 10 bytes.  Chunking and export are rv_encode_host_confluent's; the i32 overflow check of a
 * chunk counts the headers.  RV_ERR_SCHEMA: a schema without a canonical form. */
rv_status rv_encode_host_single_object(const rv_schema* s, struct ArrowArray* batch, struct ArrowSchema* batch_schema,
                                       int64_t num_chunks, rv_encoded** out);

/* One Object Container File of the batch's rows, codec "null":
 *   "Obj" 1, one metadata map block of 2 + n_meta entries: avro.schema (the exact text `s` was parsed from), avro.codec
 *   "null", then the caller's pairs in order; the 16-byte `sync` marker; then per block j: zigzag(count), zigzag(byte
 *   size), the datums of rows [j R, min((j + 1) R, n)), the sync marker (R = block_records).
 * With no rows the file ends after the header's sync marker; blocks are never empty.  The file is read back by
 * rv_decode_ocf_host.  The result holds no chunks (rv_encoded_num_chunks is 0): rv_encoded_file returns the file.
 * RV_ERR_INVALID, before any CUDA call: block_records < 1, a null sync, n_meta < 0, a metadata key that is empty,
 * starts with "avro." or repeats, a negative value length.  RV_ERR_SCHEMA, before any CUDA call: a schema whose datums
 * are always empty (records of null fields only), which no container reader takes.  RV_ERR_OVERFLOW: a block whose
 * datums exceed 2^31 - 1 bytes, with the block's first row.  The file itself may exceed 4 GiB. */
rv_status rv_encode_ocf_host(const rv_schema* s, struct ArrowArray* batch, struct ArrowSchema* batch_schema,
                             int64_t block_records, const uint8_t* sync /* 16 bytes */,
                             const char* const* meta_keys, const uint8_t* const* meta_values,
                             const int64_t* meta_value_lens, int64_t n_meta, rv_encoded** out);
/* The whole file of an rv_encode_ocf_host result: one contiguous pinned host buffer owned by `r`.  RV_ERR_INVALID for a
 * chunked result. */
rv_status rv_encoded_file(const rv_encoded* r, const uint8_t** data, int64_t* len);

/* ---- multi-GPU: gathering shard-local batches into single RecordBatches ---------------------------------------------
 * Records shard by message; each rank decodes its contiguous range (exactly the reference's per-chunk batches,
 * deserialize.rs:57-68).  When one batch over all rows is wanted (BASELINE.json configs[4]) the ranks exchange
 * rv_gather_meta_len() int64 counts each, every rank computes the same plan from them (rv_gather_plan: consecutive
 * ranks are grouped into as few batches as Arrow's i32 offsets allow), the leader of each group allocates the gathered
 * arena (rv_gather_alloc) and shares it with its group (rv_ipc_export / rv_ipc_open), and every member PUSHES its
 * buffers into it with one kernel (rv_gather_push: peer stores over NVLink, offsets rebased and bitmaps bit-shifted on
 * the way).  After a barrier the leader wraps the arena as an ordinary device-resident result (rv_gather_finish).
 * pyruhvro_b200/distributed.py drives this over torch.distributed. */
typedef struct rv_gather rv_gather;
int64_t rv_gather_meta_len(const rv_schema* s);
rv_status rv_result_gather_meta(const rv_result* r, int64_t batch, int64_t* out, int64_t cap);
rv_status rv_gather_plan(const rv_schema* s, const int64_t* metas /* [world][meta_len] */, int world, rv_gather** out);
int rv_gather_num_groups(const rv_gather* g);
int rv_gather_group_of_rank(const rv_gather* g, int rank);
/* out[0] leader rank, out[1] ranks in the group, out[2] arena bytes, out[3] rows of the gathered batch, out[4] bytes pushed by non-leaders */
rv_status rv_gather_group_info(const rv_gather* g, int group, int64_t* out5);
rv_status rv_gather_alloc(rv_gather* g, int group, void* cuda_stream, void** out_dev_ptr);
rv_status rv_gather_push(rv_gather* g, int group, int rank, rv_result* mine, int64_t batch, void* dst_base, void* cuda_stream);
rv_status rv_gather_finish(rv_gather* g, int group, rv_result** out);
void rv_gather_free(rv_gather* g);
rv_status rv_ipc_export(void* dev_ptr, uint8_t* handle64);
rv_status rv_ipc_open(const uint8_t* handle64, void** out_dev_ptr);
rv_status rv_ipc_close(void* dev_ptr);

/* Stand-alone device fix-ups (kept for callers that gather with their own collective): */
/* d_dst[i] = d_src[i] + add  — rebases a shard's i32 offsets by the totals of the shards before it. */
rv_status rv_dev_rebase_i32(int32_t* d_dst, const int32_t* d_src, int64_t n, int32_t add, void* cuda_stream);
/* ORs nbits bits of d_src_words (LSB-first) into d_dst_words starting at bit dst_bit; the destination must be
 * zero-initialised (seam words are shared between shards).  Both pointers 4-byte aligned. */
rv_status rv_dev_concat_bits(uint32_t* d_dst_words, int64_t dst_bit, const uint32_t* d_src_words, int64_t nbits, void* cuda_stream);

/* ---- memory / introspection ------------------------------------------------------------- */

void* rv_host_alloc(size_t bytes); /* pinned host memory (cudaHostAlloc); NULL on failure */
void rv_host_free(void* p);

/* Per-call timings of the calling thread's last decode, in milliseconds (CUDA events on the launch stream):
 * [0] the fused decode kernel (the pass that produced the batches), [1] an extra measuring pass (the first call on a
 * schema, or a call whose data outgrew the planned buffers; 0 otherwise), [2] unused, [3] null_count_kernel,
 * [4] H2D copy, [5] D2H copy.  Returns how many entries were written (<= cap). */
int rv_last_timings(float* out_ms, int cap);
/* Number of kernels the last decode on this thread launched. */
int rv_last_launch_count(void);
/* Passes of the fused kernel the last decode on this thread needed: 1 in steady state, 2 when it had to measure first. */
int rv_last_passes(void);
/* Drops what the schema handle learned about output sizes from earlier calls (the next call measures again). */
void rv_schema_forget_stats(const rv_schema* s);

/* Which record walker the last decode on this thread ran: "jit" (schema-specialised kernels compiled
 * with NVRTC for the device's architecture) or "interp" (the statically compiled generic kernels).
 * Both are GPU paths; RV_JIT=0 in the environment forces "interp". */
const char* rv_last_walker(void);
/* Records per tile (== threads per CTA) of the last decode on this thread: 256, or 384 where the generated walker
 * decodes a plan of more than eight streams and two 384-row CTAs fit an SM (0 before any decode). */
int rv_last_tile(void);
/* The largest tile a decode of this schema may choose: 384 for plans of more than eight streams, else 256. */
int rv_schema_max_tile(const rv_schema* s);
/* Why the schema-specialised kernels are / are not in use for this schema ("ok", the NVRTC log, ...).
 * The returned string is valid until the calling thread's next library call. */
const char* rv_schema_jit_status(const rv_schema* s);
/* Tiles of the last decode on this thread that did not fit the shared-memory windows and were walked in global
 * memory instead (slow path inside the same kernel; diagnostics). */
long long rv_last_slow_tiles(void);
/* 1 / 0: use / do not use the schema-specialised kernels from now on; -1: follow the RV_JIT environment variable. */
void rv_set_jit_enabled(int enabled);

/* The generated CUDA C++ of the schema-specialised walker (diagnostics / tests).  Returns its length;
 * copies at most cap-1 bytes + NUL into buf (buf may be NULL). */
int64_t rv_schema_walker_source(const rv_schema* s, char* buf, size_t cap);
/* The complete NVRTC source of the schema-specialised kernel for tiles of `tile` records (256, or
 * rv_schema_max_tile(s)); same buffer contract.  -1 for any other tile. */
int64_t rv_schema_kernel_source(const rv_schema* s, int tile, char* buf, size_t cap);

/* Compiles the schema-specialised kernel for `arch` (e.g. "sm_90a") at rv_schema_max_tile(s) into the on-disk
 * cubin cache (no GPU needed), so the first decode does not pay NVRTC latency. */
rv_status rv_schema_precompile(const rv_schema* s, const char* arch);

const char* rv_last_error(void);
const char* rv_version(void);

#ifdef __cplusplus
}
#endif

#endif /* RUHVRO_B200_H */
