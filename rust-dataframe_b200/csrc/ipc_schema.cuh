// ipc_schema.cuh -- what ipc.cu's flatbuffer reader gives the other host units of the library about a serialized Arrow schema.
#pragma once

#include <stddef.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/b200df.h"

namespace bdf {
// A top-level field of an Arrow schema: its name, and its temporal kind (bdf_temporal_kind, 0 for none), unit and tz.
struct ArrowField { std::string name; int kind = 0, unit = 0; bool has_tz = false; std::string tz; };
// The top-level fields of an encapsulated schema message ([0xFFFFFFFF] <int32 size> <Message flatbuffer>), as Parquet writers store it
// under ARROW:schema (the Parquet reader's Timestamp tz, parquet.cu).  False on a malformed message.
bool arrow_schema_fields(const uint8_t* p, size_t n, std::vector<ArrowField>* out);
// The encapsulated Schema message of columns (names, dtypes, temporal types or NULL), as bdf_ipc_write_typed writes it at the start of
// an IPC file: what a Parquet writer stores, base64-encoded, under ARROW:schema.
std::string arrow_schema_message(int n_cols, const char* const* names, const int32_t* dtypes, const bdf_temporal_type* types);
}  // namespace bdf
