#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include "common/fault.h"
#include "common/trace.h"
#include "common/checksum.h"
#include "common/error.h"
#include "common/json.h"
#include "common/log.h"
#include "common/mxfp8.h"
#include "common/sha256.h"
#include "common/tchash_def.h"
#include "common/yaml.h"

namespace py = pybind11;
using namespace bb;

namespace {
py::object json_to_py(const Json& j) {
  switch (j.type()) {
    case Json::Type::Null: return py::none();
    case Json::Type::Bool: return py::bool_(j.as_bool());
    case Json::Type::Int: return py::int_(j.as_int());
    case Json::Type::Double: return py::float_(j.as_double());
    case Json::Type::String: return py::str(j.as_string());
    case Json::Type::Array: {
      py::list l;
      for (const auto& e : j.as_array()) l.append(json_to_py(e));
      return l;
    }
    case Json::Type::Object: {
      py::dict d;
      for (const auto& [k, v] : j.as_object()) d[py::str(k)] = json_to_py(v);
      return d;
    }
  }
  return py::none();
}
}  // namespace

py::object bb_json_to_py(const Json& j) { return json_to_py(j); }

void bind_common(py::module_& m) {
  py::enum_<ErrorCode>(m, "ErrorCode")
      .value("OK", ErrorCode::OK)
      .value("INTERNAL_ERROR", ErrorCode::INTERNAL_ERROR)
      .value("INITIALIZATION_FAILED", ErrorCode::INITIALIZATION_FAILED)
      .value("INVALID_STATE", ErrorCode::INVALID_STATE)
      .value("OPERATION_TIMEOUT", ErrorCode::OPERATION_TIMEOUT)
      .value("RESOURCE_EXHAUSTED", ErrorCode::RESOURCE_EXHAUSTED)
      .value("NOT_IMPLEMENTED", ErrorCode::NOT_IMPLEMENTED)
      .value("INVALID_ARGUMENT", ErrorCode::INVALID_ARGUMENT)
      .value("ALREADY_EXISTS", ErrorCode::ALREADY_EXISTS)
      .value("NOT_FOUND", ErrorCode::NOT_FOUND)
      .value("BUFFER_OVERFLOW", ErrorCode::BUFFER_OVERFLOW)
      .value("OUT_OF_MEMORY", ErrorCode::OUT_OF_MEMORY)
      .value("MEMORY_POOL_NOT_FOUND", ErrorCode::MEMORY_POOL_NOT_FOUND)
      .value("MEMORY_POOL_ALREADY_EXISTS", ErrorCode::MEMORY_POOL_ALREADY_EXISTS)
      .value("INVALID_MEMORY_POOL", ErrorCode::INVALID_MEMORY_POOL)
      .value("ALLOCATION_FAILED", ErrorCode::ALLOCATION_FAILED)
      .value("INSUFFICIENT_SPACE", ErrorCode::INSUFFICIENT_SPACE)
      .value("MEMORY_ACCESS_ERROR", ErrorCode::MEMORY_ACCESS_ERROR)
      .value("IO_ERROR", ErrorCode::IO_ERROR)
      .value("NETWORK_ERROR", ErrorCode::NETWORK_ERROR)
      .value("CONNECTION_FAILED", ErrorCode::CONNECTION_FAILED)
      .value("TRANSFER_FAILED", ErrorCode::TRANSFER_FAILED)
      .value("UCX_ERROR", ErrorCode::UCX_ERROR)
      .value("INVALID_ADDRESS", ErrorCode::INVALID_ADDRESS)
      .value("REMOTE_ENDPOINT_ERROR", ErrorCode::REMOTE_ENDPOINT_ERROR)
      .value("RPC_FAILED", ErrorCode::RPC_FAILED)
      .value("FABRIC_ERROR", ErrorCode::FABRIC_ERROR)
      .value("ETCD_ERROR", ErrorCode::ETCD_ERROR)
      .value("ETCD_KEY_NOT_FOUND", ErrorCode::ETCD_KEY_NOT_FOUND)
      .value("ETCD_TRANSACTION_FAILED", ErrorCode::ETCD_TRANSACTION_FAILED)
      .value("ETCD_LEASE_ERROR", ErrorCode::ETCD_LEASE_ERROR)
      .value("ETCD_WATCH_ERROR", ErrorCode::ETCD_WATCH_ERROR)
      .value("LEADER_ELECTION_FAILED", ErrorCode::LEADER_ELECTION_FAILED)
      .value("SERVICE_REGISTRATION_FAILED", ErrorCode::SERVICE_REGISTRATION_FAILED)
      .value("NOT_LEADER", ErrorCode::NOT_LEADER)
      .value("OBJECT_NOT_FOUND", ErrorCode::OBJECT_NOT_FOUND)
      .value("OBJECT_ALREADY_EXISTS", ErrorCode::OBJECT_ALREADY_EXISTS)
      .value("INVALID_KEY", ErrorCode::INVALID_KEY)
      .value("INVALID_WORKER", ErrorCode::INVALID_WORKER)
      .value("WORKER_NOT_READY", ErrorCode::WORKER_NOT_READY)
      .value("NO_COMPLETE_WORKER", ErrorCode::NO_COMPLETE_WORKER)
      .value("DATA_CORRUPTION", ErrorCode::DATA_CORRUPTION)
      .value("CHECKSUM_MISMATCH", ErrorCode::CHECKSUM_MISMATCH)
      .value("OBJECT_NOT_READY", ErrorCode::OBJECT_NOT_READY)
      .value("CLIENT_ERROR", ErrorCode::CLIENT_ERROR)
      .value("CLIENT_NOT_FOUND", ErrorCode::CLIENT_NOT_FOUND)
      .value("CLIENT_ALREADY_EXISTS", ErrorCode::CLIENT_ALREADY_EXISTS)
      .value("CLIENT_DISCONNECTED", ErrorCode::CLIENT_DISCONNECTED)
      .value("SESSION_EXPIRED", ErrorCode::SESSION_EXPIRED)
      .value("INVALID_CLIENT_STATE", ErrorCode::INVALID_CLIENT_STATE)
      .value("ACCESS_DENIED", ErrorCode::ACCESS_DENIED)
      .value("QUOTA_EXCEEDED", ErrorCode::QUOTA_EXCEEDED)
      .value("CONFIG_ERROR", ErrorCode::CONFIG_ERROR)
      .value("INVALID_CONFIGURATION", ErrorCode::INVALID_CONFIGURATION)
      .value("INVALID_PARAMETERS", ErrorCode::INVALID_PARAMETERS)
      .value("MISSING_REQUIRED_FIELD", ErrorCode::MISSING_REQUIRED_FIELD)
      .value("VALUE_OUT_OF_RANGE", ErrorCode::VALUE_OUT_OF_RANGE);
  m.def("error_string", [](ErrorCode c) { return std::string(to_string(c)); });
  m.def("error_description", [](ErrorCode c) { return std::string(get_error_description(c)); });
  m.def("error_domain", [](ErrorCode c) { return std::string(to_string(get_error_domain(c))); });

  py::enum_<ChecksumAlgo>(m, "ChecksumAlgo")
      .value("NONE", ChecksumAlgo::NONE)
      .value("CRC32C", ChecksumAlgo::CRC32C)
      .value("BBH64", ChecksumAlgo::BBH64)
      .value("XXH3", ChecksumAlgo::XXH3);

  m.def("crc32c", [](py::buffer b, uint32_t crc) {
    py::buffer_info i = b.request();
    return crc32c(i.ptr, static_cast<size_t>(i.size * i.itemsize), crc);
  }, py::arg("data"), py::arg("crc") = 0);
  m.def("crc32c_sw", [](py::buffer b, uint32_t crc) {
    py::buffer_info i = b.request();
    return crc32c_sw(i.ptr, static_cast<size_t>(i.size * i.itemsize), crc);
  }, py::arg("data"), py::arg("crc") = 0);
  m.def("crc32c_raw", [](py::buffer b, uint32_t rem) {
    py::buffer_info i = b.request();
    return crc32c_raw(i.ptr, static_cast<size_t>(i.size * i.itemsize), rem);
  }, py::arg("data"), py::arg("rem") = 0);
  m.def("crc32c_combine", &crc32c_combine);
  m.def("crc32c_from_raw", &crc32c_from_raw);
  m.def("crc32c_hw_available", &crc32c_hw_available);
  m.def("gf2_mulmod", &gf2_mulmod);
  m.def("gf2_xpow_bytes", &gf2_xpow_bytes);
  m.def("bbh64", [](py::buffer b) {
    py::buffer_info i = b.request();
    return bbh64(i.ptr, static_cast<size_t>(i.size * i.itemsize));
  });
  m.def("xxh3t64", [](py::buffer b) {
    py::buffer_info i = b.request();
    return xxh3t64(i.ptr, static_cast<size_t>(i.size * i.itemsize));
  }, "Tiled XXH3: the standard XXH3-64 of every 16 KiB tile (last one zero padded), combined order-independently.");
  m.def("xxh3_tile", [](py::buffer b) {
    py::buffer_info i = b.request();
    if (i.size * i.itemsize != 16384) throw py::value_error("xxh3_tile wants exactly 16384 bytes");
    return xxh3_tile(i.ptr);
  }, "XXH3_64bits() of one 16 KiB tile (default secret, seed 0) -- equals xxhash.xxh3_64_intdigest(tile).");
  m.def("xxh3t64_partial", [](py::buffer b, uint64_t first_tile, uint64_t ntiles) {
    py::buffer_info i = b.request();
    return xxh3t64_partial(i.ptr, static_cast<size_t>(i.size * i.itemsize), first_tile, ntiles);
  });
  m.def("bbh64_reference", [](py::buffer b) {
    py::buffer_info i = b.request();
    return bbh64_reference(i.ptr, static_cast<size_t>(i.size * i.itemsize));
  });
  m.def("bbh64_using", [](const std::string& impl, py::buffer b) -> py::object {
    py::buffer_info i = b.request();
    bool ok = false;
    const uint64_t d = bbh64_using(impl, i.ptr, static_cast<size_t>(i.size * i.itemsize), &ok);
    if (!ok) return py::none();
    return py::int_(d);
  });
  m.def("bbh64_partial", [](py::buffer b, uint64_t first_tile, uint64_t ntiles) {
    py::buffer_info i = b.request();
    return bbh64_partial(i.ptr, static_cast<size_t>(i.size * i.itemsize), first_tile, ntiles);
  });
  m.def("bbh64_finalize", &bbh64_finalize);
  m.def("bbh64_impl_name", [] { return std::string(bbh64_impl_name()); });
  m.def("sha256", [](py::bytes b) {
    const std::string s = b;
    const Sha256Digest d = sha256(s);
    return py::bytes(reinterpret_cast<const char*>(d.data()), d.size());
  });
  m.def("hmac_sha256", [](py::bytes key, py::bytes msg) {
    const std::string k = key, v = msg;
    const Sha256Digest d = hmac_sha256(k, v);
    return py::bytes(reinterpret_cast<const char*>(d.data()), d.size());
  });
  m.def("bbh64_weight", [](uint32_t k, uint32_t n) { return tchash::weight(k, n); });
  m.def("bbh64_off_to_row", [](uint32_t o) { return tchash::off_to_row(o); });
  m.def("bbh64_off_to_k", [](uint32_t o) { return tchash::off_to_k(o); });

  m.def("parse_yaml", [](const std::string& text) -> py::object {
    std::string err;
    auto j = parse_yaml(text, &err);
    if (!j) throw py::value_error("yaml: " + err);
    return json_to_py(*j);
  });
  m.def("parse_json", [](const std::string& text) -> py::object {
    std::string err;
    auto j = Json::parse(text, &err);
    if (!j) throw py::value_error("json: " + err);
    return json_to_py(*j);
  });
  m.def("json_roundtrip", [](const std::string& text) {
    std::string err;
    auto j = Json::parse(text, &err);
    if (!j) throw py::value_error("json: " + err);
    return j->dump();
  });
  // tracing + fault injection (csrc/common/trace.h, fault.h)
  m.def("trace_enable", [](bool on, size_t cap) { trace::enable(on, cap); }, py::arg("on") = true, py::arg("ring_capacity") = size_t{1} << 16);
  m.def("trace_enabled", &trace::enabled);
  m.def("trace_dump", &trace::dump, "writes Chrome/Perfetto traceEvents JSON; returns the number of events");
  m.def("trace_recorded", &trace::recorded);
  m.def("trace_clear", &trace::clear);
  m.def("fault_arm", &fault::arm, py::arg("name"), py::arg("value") = 1, py::arg("count") = -1);
  m.def("fault_disarm", &fault::disarm);
  m.def("fault_clear", &fault::clear);
  m.def("fault_arm_from_spec", &fault::arm_from_spec);
  m.def("parse_size", [](const std::string& s) -> py::object {
    auto v = parse_size(s);
    if (!v) return py::none();
    return py::int_(*v);
  });
  py::enum_<mxfp8::Wide>(m, "MxWide", "Element type of the wide (unpacked) side of an MXFP8 transfer")
      .value("BF16", mxfp8::Wide::BF16)
      .value("F16", mxfp8::Wide::F16)
      .value("F32", mxfp8::Wide::F32);
  m.def("mxfp8_wide_bytes", [](mxfp8::Wide w) { return mxfp8::wide_bytes(w); });
  m.def("mxfp8_pack_ref", [](py::buffer wide_bits, mxfp8::Wide wide) {
    py::buffer_info i = wide_bits.request();
    const size_t n = static_cast<size_t>(i.size * i.itemsize) / mxfp8::wide_bytes(wide);
    if (n % 32) throw py::value_error("element count must be a multiple of 32");
    std::string out(mxfp8::packed_bytes(n), '\0');
    mxfp8::pack(i.ptr, wide, n, reinterpret_cast<uint8_t*>(out.data()));
    return py::bytes(out);
  }, py::arg("wide_bits"), py::arg("wide") = mxfp8::Wide::BF16,
     "CPU reference: raw bits of n elements of type `wide` (bf16 / fp16 / fp32) -> [E4M3 payload | E8M0 scales]");
  m.def("mxfp8_unpack_ref", [](py::buffer packed, size_t n, mxfp8::Wide wide) {
    py::buffer_info i = packed.request();
    if (static_cast<size_t>(i.size * i.itemsize) < mxfp8::packed_bytes(n)) throw py::value_error("packed buffer too small");
    std::string out(n * mxfp8::wide_bytes(wide), '\0');
    mxfp8::unpack(static_cast<const uint8_t*>(i.ptr), n, wide, out.data());
    return py::bytes(out);
  }, py::arg("packed"), py::arg("n"), py::arg("wide") = mxfp8::Wide::BF16,
     "CPU reference: packed object of n elements -> raw bits of n elements of type `wide`");
  m.def("e4m3_from_float", [](float f) { return mxfp8::float_to_e4m3_sat(f); });
  m.def("e4m3_to_float", [](uint8_t v) { return mxfp8::e4m3_to_float(v); });
  m.def("mxfp8_packed_bytes", [](size_t n) { return mxfp8::packed_bytes(n); });
  m.def("set_log_level", [](int l) { set_log_level(static_cast<LogLevel>(l)); });
}
