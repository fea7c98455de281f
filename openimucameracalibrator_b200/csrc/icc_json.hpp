// Minimal JSON + UBJSON value, reader and writer for the drop-in CLI (no third-party dependency is available offline).
//
// Covers exactly what the reference's hot CLI reads and writes through nlohmann::json:
//   text JSON      src/io/read_camera_calibration.cc:35-119, read_telemetry.cc:29-69, read_misc.cc:30-150
//   UBJSON corners src/io/read_scene.cc:25-41 (nlohmann::json::from_ubjson of BoardExtractor's output)
//   result JSON    applications/continuous_time_imu_to_camera_calibration.cc:247-332 (std::setw(4), keys sorted like std::map)
#pragma once
#include <charconv>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <map>
#include <memory>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>

namespace iccjson {

struct Value;
using Object = std::map<std::string, Value>;   // sorted keys, like nlohmann::json's default object_t
using Array = std::vector<Value>;

struct Value {
  enum Type : uint8_t { Null, Bool, Int, Float, String, Arr, Obj } type = Null;
  union { bool b; int64_t i; double d; };                 // scalar payload (most values of a telemetry / corner file are numbers)
  std::shared_ptr<std::string> sp;                          // String
  std::shared_ptr<Array> a;
  std::shared_ptr<Object> o;

  Value() : i(0) {}
  Value(bool v) : type(Bool), i(0) { b = v; }
  Value(int v) : type(Int), i(v) {}
  Value(int64_t v) : type(Int), i(v) {}
  Value(double v) : type(Float), d(v) {}
  Value(const char* v) : type(String), i(0), sp(std::make_shared<std::string>(v)) {}
  Value(const std::string& v) : type(String), i(0), sp(std::make_shared<std::string>(v)) {}
  Value(std::string&& v) : type(String), i(0), sp(std::make_shared<std::string>(std::move(v))) {}
  static Value array() { Value v; v.type = Arr; v.a = std::make_shared<Array>(); return v; }
  static Value object() { Value v; v.type = Obj; v.o = std::make_shared<Object>(); return v; }

  bool is_object() const { return type == Obj; }
  bool is_array() const { return type == Arr; }
  bool is_number() const { return type == Int || type == Float; }
  bool contains(const std::string& k) const { return type == Obj && o->count(k); }
  size_t size() const { return type == Arr ? a->size() : type == Obj ? o->size() : 0; }
  double num() const { if (type == Int) return double(i); if (type == Float) return d; throw std::runtime_error("json: value is not a number"); }
  int64_t integer() const { if (type == Int) return i; if (type == Float) return int64_t(d); throw std::runtime_error("json: value is not a number"); }
  const std::string& str() const { if (type != String) throw std::runtime_error("json: value is not a string"); return *sp; }
  const Value& at(const std::string& k) const { if (type == Obj) { const auto it = o->find(k); if (it != o->end()) return it->second; } throw std::runtime_error("json: missing key '" + k + "'"); }
  const Value& at(size_t k) const { if (type != Arr || k >= a->size()) throw std::runtime_error("json: array index out of range"); return (*a)[k]; }
  Value& operator[](const std::string& k) { if (type == Null) { type = Obj; o = std::make_shared<Object>(); } if (type != Obj) throw std::runtime_error("json: not an object"); return (*o)[k]; }
  void push_back(const Value& v) { if (type == Null) { type = Arr; a = std::make_shared<Array>(); } a->push_back(v); }
};

// ---- text JSON ----------------------------------------------------------------------------------------------------
class TextParser {
 public:
  explicit TextParser(const std::string& t) : t_(t) {}
  Value parse() { Value v = value(); ws(); if (p_ != t_.size()) fail("trailing characters"); return v; }
 protected:
  const std::string& t_; size_t p_ = 0;
  [[noreturn]] void fail(const std::string& m) { throw std::runtime_error("json parse error at byte " + std::to_string(p_) + ": " + m); }
  void ws() { while (p_ < t_.size() && (t_[p_] == ' ' || t_[p_] == '\n' || t_[p_] == '\t' || t_[p_] == '\r')) ++p_; }
  Value value() {
    ws(); if (p_ >= t_.size()) fail("unexpected end");
    const char c = t_[p_];
    if (c == '{') return object();
    if (c == '[') return array();
    if (c == '"') return Value(string());
    if (!t_.compare(p_, 4, "true")) { p_ += 4; return Value(true); }
    if (!t_.compare(p_, 5, "false")) { p_ += 5; return Value(false); }
    if (!t_.compare(p_, 4, "null")) { p_ += 4; return Value(); }
    if (!t_.compare(p_, 3, "NaN")) { p_ += 3; return Value(std::nan("")); }
    return number();
  }
  Value object() {
    Value v = Value::object(); ++p_; ws();
    if (p_ < t_.size() && t_[p_] == '}') { ++p_; return v; }
    for (;;) {
      ws(); if (p_ >= t_.size() || t_[p_] != '"') fail("expected key");
      std::string k = string(); ws();
      if (p_ >= t_.size() || t_[p_] != ':') fail("expected ':'");
      ++p_; v.o->insert_or_assign(v.o->end(), std::move(k), value()); ws();
      if (p_ < t_.size() && t_[p_] == ',') { ++p_; continue; }
      if (p_ < t_.size() && t_[p_] == '}') { ++p_; return v; }
      fail("expected ',' or '}'");
    }
  }
  Value array() {
    Value v = Value::array(); ++p_; ws();
    if (p_ < t_.size() && t_[p_] == ']') { ++p_; return v; }
    for (;;) {
      v.a->push_back(value()); ws();
      if (p_ < t_.size() && t_[p_] == ',') { ++p_; continue; }
      if (p_ < t_.size() && t_[p_] == ']') { ++p_; return v; }
      fail("expected ',' or ']'");
    }
  }
  std::string string() {
    std::string out; ++p_;
    while (p_ < t_.size() && t_[p_] != '"') {
      char c = t_[p_++];
      if (c == '\\') {
        if (p_ >= t_.size()) fail("bad escape");
        const char e = t_[p_++];
        switch (e) { case 'n': out += '\n'; break; case 't': out += '\t'; break; case 'r': out += '\r'; break; case 'b': out += '\b'; break; case 'f': out += '\f'; break;
          case 'u': { if (p_ + 4 > t_.size()) fail("bad \\u"); unsigned cp = std::stoul(t_.substr(p_, 4), nullptr, 16); p_ += 4; if (cp < 0x80) out += char(cp); else if (cp < 0x800) { out += char(0xC0 | (cp >> 6)); out += char(0x80 | (cp & 0x3F)); } else { out += char(0xE0 | (cp >> 12)); out += char(0x80 | ((cp >> 6) & 0x3F)); out += char(0x80 | (cp & 0x3F)); } break; }
          default: out += e; }
      } else out += c;
    }
    if (p_ >= t_.size()) fail("unterminated string");
    ++p_; return out;
  }
  Value number() {
    const size_t s = p_; bool is_float = false;
    if (p_ < t_.size() && (t_[p_] == '-' || t_[p_] == '+')) ++p_;
    while (p_ < t_.size() && (isdigit((unsigned char)t_[p_]) || t_[p_] == '.' || t_[p_] == 'e' || t_[p_] == 'E' || t_[p_] == '-' || t_[p_] == '+')) { if (t_[p_] == '.' || t_[p_] == 'e' || t_[p_] == 'E') is_float = true; ++p_; }
    if (p_ == s) fail("unexpected character");
    const char* first = t_.data() + s + (t_[s] == '+' ? 1 : 0); const char* last = t_.data() + p_;
    if (!is_float) { int64_t iv = 0; const auto r = std::from_chars(first, last, iv); if (r.ec == std::errc() && r.ptr == last) return Value(iv); }
    double dv = 0.0; const auto r = std::from_chars(first, last, dv);
    if (r.ec == std::errc() && r.ptr == last) return Value(dv);
    return Value(std::stod(std::string(first, last)));      // out-of-range literals etc.: the C library decides, as before
  }
};

inline std::string read_file(const std::string& path, bool binary = false) {
  std::ifstream f(path, binary ? std::ios::binary : std::ios::in);
  if (!f.is_open()) throw std::runtime_error("could not open " + path);
  f.seekg(0, std::ios::end); const std::streamoff n = f.tellg(); f.seekg(0, std::ios::beg);
  std::string out;
  if (n > 0) { out.resize((size_t)n); f.read(&out[0], n); out.resize((size_t)f.gcount()); }
  else { std::stringstream ss; ss << f.rdbuf(); out = ss.str(); }   // not seekable
  return out;
}
inline Value parse_text(const std::string& text) { return TextParser(text).parse(); }
inline Value load_json(const std::string& path) { return parse_text(read_file(path)); }

inline std::string number_to_string(double v) {
  if (!std::isfinite(v)) return "null";   // nlohmann dumps non-finite numbers as null
  char buf[64]; auto r = std::to_chars(buf, buf + sizeof buf, v); std::string s(buf, r.ptr);
  if (s.find_first_of(".eEn") == std::string::npos) s += ".0";
  return s;
}
// Streaming writer with nlohmann::json::dump(indent) formatting: objects / arrays one member per line, "key": value, "{}" / "[]" when
// empty.  dump(Value) below walks a tree through it; the CLI streams the (large) trajectory object through the same code without
// building a tree, so both routes produce identical bytes.  With a FILE* sink the text is flushed in ~1 MB pieces.
class Writer {
 public:
  explicit Writer(int indent, std::string* sink) : indent_(indent), str_(sink) {}
  // a writer that continues INSIDE open containers: `members[d]` = members already written in the container at depth d (fragments
  // produced this way concatenate to exactly the bytes one writer would have produced)
  Writer(int indent, std::string* sink, const std::vector<size_t>& members) : indent_(indent), str_(sink), count_(members) {}
  Writer(int indent, FILE* sink) : indent_(indent), file_(sink) { buf_.reserve(size_t(1) << 21); }
  ~Writer() { flush(); }
  void begin_object() { open('{'); }
  void end_object() { close('}'); }
  void begin_array() { open('['); }
  void end_array() { close(']'); }
  void key(const std::string& k) { member(); out() += '"'; out() += k; out() += "\": "; after_key_ = true; }
  void value(double v) { element(); number(v); }
  void value(int64_t v) { element(); char b[32]; const auto r = std::to_chars(b, b + sizeof b, v); out().append(b, r.ptr); }
  void value(bool v) { element(); out() += v ? "true" : "false"; }
  void null() { element(); out() += "null"; }
  void value(const std::string& v) { element(); string(v); }
  void value(const Value& v) {
    switch (v.type) {
      case Value::Null: null(); break;
      case Value::Bool: value(v.b); break;
      case Value::Int: value(v.i); break;
      case Value::Float: value(v.d); break;
      case Value::String: value(*v.sp); break;
      case Value::Arr: begin_array(); for (const Value& e : *v.a) value(e); end_array(); break;
      case Value::Obj: begin_object(); for (const auto& kv : *v.o) { key(kv.first); value(kv.second); } end_object(); break;
    }
  }
  // pre-formatted members of the innermost open container (see the fragment constructor)
  void raw_members(const std::string& text, size_t n_members) { if (n_members == 0) return; if (file_) { flush(); fwrite(text.data(), 1, text.size(), file_); } else out() += text; count_.back() += n_members; }
  void flush() { if (file_ && !buf_.empty()) { fwrite(buf_.data(), 1, buf_.size(), file_); buf_.clear(); } }
 private:
  int indent_; std::string* str_ = nullptr; FILE* file_ = nullptr; std::string buf_;
  std::vector<size_t> count_;   // members written so far, per open container
  bool after_key_ = false;
  std::string& out() { return str_ ? *str_ : buf_; }
  void newline(size_t depth) { out() += '\n'; out().append(indent_ * depth, ' '); if (file_ && buf_.size() > (size_t(1) << 20)) flush(); }
  void member() { if (!count_.empty()) { if (count_.back()++) out() += ','; newline(count_.size()); } }
  void element() { if (after_key_) after_key_ = false; else member(); }     // a value after key() continues the line; array elements start one
  void open(char c) { element(); out() += c; count_.push_back(0); }
  void close(char c) { const size_t n = count_.back(); count_.pop_back(); if (n) newline(count_.size()); out() += c; }
  void number(double v) {
    if (!std::isfinite(v)) { out() += "null"; return; }   // nlohmann dumps non-finite numbers as null
    char b[64]; const auto r = std::to_chars(b, b + sizeof b, v);
    bool plain = true; for (const char* p = b; p != r.ptr; ++p) if (*p == '.' || *p == 'e' || *p == 'E' || *p == 'n') { plain = false; break; }
    out().append(b, r.ptr); if (plain) out() += ".0";
  }
  void string(const std::string& v) { out() += '"'; for (char c : v) { if (c == '"' || c == '\\') { out() += '\\'; out() += c; } else if (c == '\n') out() += "\\n"; else out() += c; } out() += '"'; }
};
inline std::string dump(const Value& v, int indent = 4) { std::string s; { Writer w(indent, &s); w.value(v); } return s; }

// ---- UBJSON (draft 12) --------------------------------------------------------------------------------------------
class UbjsonParser {
 public:
  explicit UbjsonParser(const std::string& d) : d_(d) {}
  Value parse() { return value(next()); }
 protected:
  const std::string& d_; size_t p_ = 0;
  [[noreturn]] void fail(const std::string& m) { throw std::runtime_error("ubjson parse error at byte " + std::to_string(p_) + ": " + m); }
  unsigned char next() { if (p_ >= d_.size()) fail("unexpected end"); return (unsigned char)d_[p_++]; }
  unsigned char peek() { if (p_ >= d_.size()) fail("unexpected end"); return (unsigned char)d_[p_]; }
  template <class T> T be() { if (p_ + sizeof(T) > d_.size()) fail("unexpected end"); unsigned char b[sizeof(T)]; for (size_t k = 0; k < sizeof(T); ++k) b[sizeof(T) - 1 - k] = (unsigned char)d_[p_ + k]; p_ += sizeof(T); T v; memcpy(&v, b, sizeof(T)); return v; }
  int64_t integer(unsigned char t) {
    switch (t) { case 'i': return be<int8_t>(); case 'U': return be<uint8_t>(); case 'I': return be<int16_t>(); case 'l': return be<int32_t>(); case 'L': return be<int64_t>();
      case 'u': return be<uint16_t>(); case 'm': return be<uint32_t>(); case 'M': return (int64_t)be<uint64_t>(); default: fail("expected integer type"); }
  }
  std::string raw_string() { const int64_t n = integer(next()); if (n < 0 || p_ + (size_t)n > d_.size()) fail("bad string length"); std::string s = d_.substr(p_, (size_t)n); p_ += (size_t)n; return s; }
  Value value(unsigned char t) {
    switch (t) {
      case 'Z': return Value(); case 'T': return Value(true); case 'F': return Value(false); case 'N': return value(next());
      case 'i': case 'U': case 'I': case 'l': case 'L': case 'u': case 'm': case 'M': return Value(integer(t));
      case 'd': return Value(double(be<float>())); case 'D': return Value(be<double>());
      case 'C': return Value(std::string(1, (char)next())); case 'S': return Value(raw_string());
      case 'H': { std::string s = raw_string(); return Value(std::stod(s)); }
      case '[': {
        Value v = Value::array(); unsigned char et = 0; int64_t n = -1;
        if (peek() == '$') { ++p_; et = next(); if (next() != '#') fail("expected '#' after '$'"); n = integer(next()); }
        else if (peek() == '#') { ++p_; n = integer(next()); }
        if (n >= 0) { for (int64_t k = 0; k < n; ++k) v.a->push_back(value(et ? et : next())); }
        else { while (peek() != ']') v.a->push_back(value(next())); ++p_; }
        return v; }
      case '{': {
        Value v = Value::object(); unsigned char et = 0; int64_t n = -1;
        if (peek() == '$') { ++p_; et = next(); if (next() != '#') fail("expected '#' after '$'"); n = integer(next()); }
        else if (peek() == '#') { ++p_; n = integer(next()); }
        if (n >= 0) { for (int64_t k = 0; k < n; ++k) { std::string key = raw_string(); v.o->insert_or_assign(v.o->end(), std::move(key), value(et ? et : next())); } }
        else { while (peek() != '}') { std::string key = raw_string(); v.o->insert_or_assign(v.o->end(), std::move(key), value(next())); } ++p_; }
        return v; }
      default: fail(std::string("unknown type marker '") + (char)t + "'");
    }
  }
};
inline Value load_ubjson(const std::string& path) { const std::string d = read_file(path, true); return UbjsonParser(d).parse(); }

// nlohmann::json::to_ubjson(j) with its defaults (no count or type optimisation): keys in std::map order, every floating-point number as
// 'D' (big-endian double), every integer in the smallest of i, U, I, l, L that holds it, strings and keys with such a length prefix.
class UbjsonWriter {
 public:
  static std::string dump(const Value& v) { std::string s; write(s, v); return s; }
  static void write(std::string& out, const Value& v) {
    switch (v.type) {
      case Value::Null: out += 'Z'; break;
      case Value::Bool: out += v.b ? 'T' : 'F'; break;
      case Value::Int: integer(out, v.i); break;
      case Value::Float: out += 'D'; be(out, v.d); break;
      case Value::String: out += 'S'; string(out, *v.sp); break;
      case Value::Arr: out += '['; for (const Value& e : *v.a) write(out, e); out += ']'; break;
      case Value::Obj: out += '{'; for (const auto& kv : *v.o) { string(out, kv.first); write(out, kv.second); } out += '}'; break;
    }
  }
 private:
  template <class T> static void be(std::string& out, T v) { unsigned char b[sizeof(T)]; memcpy(b, &v, sizeof(T)); for (size_t k = 0; k < sizeof(T); ++k) out += (char)b[sizeof(T) - 1 - k]; }
  static void integer(std::string& out, int64_t n) {
    if (n >= INT8_MIN && n <= INT8_MAX) { out += 'i'; be(out, (int8_t)n); }
    else if (n >= 0 && n <= UINT8_MAX) { out += 'U'; be(out, (uint8_t)n); }
    else if (n >= INT16_MIN && n <= INT16_MAX) { out += 'I'; be(out, (int16_t)n); }
    else if (n >= INT32_MIN && n <= INT32_MAX) { out += 'l'; be(out, (int32_t)n); }
    else { out += 'L'; be(out, n); }
  }
  static void string(std::string& out, const std::string& s) { integer(out, (int64_t)s.size()); out += s; }
};
inline std::string dump_ubjson(const Value& v) { return UbjsonWriter::dump(v); }

}  // namespace iccjson
