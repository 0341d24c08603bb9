// pcd_io.h — PCD (Point Cloud Data v0.7) reader/writer for the front end of the `b200_integrate` program.
//
// The reference loads its inputs with pcl::io::loadPCDFile into pcl::PointXYZRGBA (src/prog/integrate.cpp:548).
// PCL is not a dependency here; this reads the three DATA encodings PCL writes (ascii, binary,
// binary_compressed = LZF over a structure-of-arrays layout) and maps the fields x, y, z and rgb/rgba
// onto a 16-byte point {x, y, z, b, g, r, a}.  Fields the file lacks keep PointXYZRGBA's defaults
// (colour 0,0,0 with alpha 255); other fields are ignored, as loadPCDFile's field mapping does.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <limits>
#include <sstream>
#include <string>
#include <vector>

namespace b200prog {

struct PointXYZRGBA16 { float x, y, z; std::uint8_t b, g, r, a; };
static_assert (sizeof (PointXYZRGBA16) == 16, "layout");

struct Cloud
{
  std::vector<PointXYZRGBA16> points;
  std::uint32_t width = 0, height = 0;
  bool has_color = false;
  std::size_t size () const { return points.size (); }
};

// liblzf decompression (the format PCL's binary_compressed uses): control byte < 32 = literal run of ctrl+1
// bytes; otherwise a back reference of length (ctrl >> 5) + 2 (+ next byte when the 3-bit length is 7) at
// distance ((ctrl & 31) << 8 | next byte) + 1.
inline bool lzf_decompress (const unsigned char* in, std::size_t in_len, unsigned char* out, std::size_t out_len)
{
  const unsigned char *ip = in, *in_end = in + in_len;
  unsigned char *op = out, *out_end = out + out_len;
  while (ip < in_end)
  {
    unsigned ctrl = *ip++;
    if (ctrl < 32)
    {
      ++ctrl;
      if (op + ctrl > out_end || ip + ctrl > in_end) return false;
      std::memcpy (op, ip, ctrl); op += ctrl; ip += ctrl;
    }
    else
    {
      unsigned len = ctrl >> 5;
      if (ip >= in_end) return false;
      if (len == 7) { len += *ip++; if (ip >= in_end) return false; }
      std::ptrdiff_t dist = (std::ptrdiff_t) (((ctrl & 0x1f) << 8) | *ip++) + 1;
      len += 2;
      if (op - out < dist || op + len > out_end) return false;
      const unsigned char* ref = op - dist;
      for (unsigned i = 0; i < len; ++i) *op++ = *ref++;          // may overlap: byte by byte
    }
  }
  return op == out_end;
}

// a (valid, uncompressed) LZF stream: literal runs only.  Enough for the writer below and for tests.
inline std::vector<unsigned char> lzf_store (const unsigned char* in, std::size_t n)
{
  std::vector<unsigned char> out;
  out.reserve (n + n / 32 + 1);
  for (std::size_t i = 0; i < n; i += 32)
  {
    std::size_t run = n - i < 32 ? n - i : 32;
    out.push_back ((unsigned char) (run - 1));
    out.insert (out.end (), in + i, in + i + run);
  }
  return out;
}

namespace detail {
struct Field { std::string name; int size = 4; char type = 'F'; int count = 1; std::size_t offset = 0; };

inline double scalar_from (const unsigned char* p, const Field& f)
{
  switch (f.type)
  {
    case 'F': if (f.size == 4) { float v; std::memcpy (&v, p, 4); return v; } else { double v; std::memcpy (&v, p, 8); return v; }
    case 'I': switch (f.size) { case 1: { std::int8_t v; std::memcpy (&v, p, 1); return v; } case 2: { std::int16_t v; std::memcpy (&v, p, 2); return v; }
                                case 4: { std::int32_t v; std::memcpy (&v, p, 4); return v; } default: { std::int64_t v; std::memcpy (&v, p, 8); return (double) v; } }
    default:  switch (f.size) { case 1: { std::uint8_t v; std::memcpy (&v, p, 1); return v; } case 2: { std::uint16_t v; std::memcpy (&v, p, 2); return v; }
                                case 4: { std::uint32_t v; std::memcpy (&v, p, 4); return v; } default: { std::uint64_t v; std::memcpy (&v, p, 8); return (double) v; } }
  }
}
// ascii token -> the field's binary representation
inline void token_to_bytes (const std::string& tok, const Field& f, unsigned char* p)
{
  if (f.type == 'F')
  {
    double v = (tok == "nan" || tok == "NaN" || tok == "-nan") ? std::numeric_limits<double>::quiet_NaN () : std::strtod (tok.c_str (), nullptr);
    if (f.size == 4) { float w = (float) v; std::memcpy (p, &w, 4); } else std::memcpy (p, &v, 8);
  }
  else if (f.type == 'I') { long long v = std::strtoll (tok.c_str (), nullptr, 10); std::memcpy (p, &v, f.size); }     // little endian
  else { unsigned long long v = std::strtoull (tok.c_str (), nullptr, 10); std::memcpy (p, &v, f.size); }
}
} // namespace detail

// Returns an empty string on success, else what went wrong.
inline std::string load_pcd (const std::string& path, Cloud& cloud)
{
  using detail::Field;
  std::ifstream f (path, std::ios::binary);
  if (!f) return "cannot open " + path;
  std::vector<Field> fields;
  std::size_t npoints = 0; bool have_points = false;
  std::string data_mode, line;
  cloud = Cloud ();
  while (std::getline (f, line))
  {
    if (!line.empty () && line.back () == '\r') line.pop_back ();
    if (line.empty () || line[0] == '#') continue;
    std::istringstream ls (line);
    std::string key; ls >> key;
    std::vector<std::string> v; for (std::string t; ls >> t;) v.push_back (t);
    if (key == "VERSION" || key == "VIEWPOINT") continue;
    else if (key == "FIELDS" || key == "COLUMNS") { fields.resize (v.size ()); for (std::size_t i = 0; i < v.size (); ++i) fields[i].name = v[i]; }
    else if (key == "SIZE") { if (v.size () != fields.size ()) return "SIZE/FIELDS mismatch"; for (std::size_t i = 0; i < v.size (); ++i) fields[i].size = std::atoi (v[i].c_str ()); }
    else if (key == "TYPE") { if (v.size () != fields.size ()) return "TYPE/FIELDS mismatch"; for (std::size_t i = 0; i < v.size (); ++i) fields[i].type = v[i][0]; }
    else if (key == "COUNT") { if (v.size () != fields.size ()) return "COUNT/FIELDS mismatch"; for (std::size_t i = 0; i < v.size (); ++i) fields[i].count = std::atoi (v[i].c_str ()); }
    else if (key == "WIDTH" && !v.empty ()) cloud.width = (std::uint32_t) std::strtoul (v[0].c_str (), nullptr, 10);
    else if (key == "HEIGHT" && !v.empty ()) cloud.height = (std::uint32_t) std::strtoul (v[0].c_str (), nullptr, 10);
    else if (key == "POINTS" && !v.empty ()) { npoints = std::strtoull (v[0].c_str (), nullptr, 10); have_points = true; }
    else if (key == "DATA" && !v.empty ()) { data_mode = v[0]; break; }
    else return "unexpected header line: " + line;
  }
  if (data_mode.empty () || fields.empty ()) return "not a PCD file (no FIELDS/DATA): " + path;
  if (!have_points) npoints = (std::size_t) cloud.width * cloud.height;
  if (cloud.height == 0) { cloud.height = 1; cloud.width = (std::uint32_t) npoints; }
  std::size_t rec = 0;
  for (auto& fd : fields)
  {
    if (fd.size != 1 && fd.size != 2 && fd.size != 4 && fd.size != 8) return "unsupported field size";
    if (fd.count < 1) fd.count = 1;
    fd.offset = rec; rec += (std::size_t) fd.size * fd.count;
  }
  int fx = -1, fy = -1, fz = -1, fc = -1;
  for (std::size_t i = 0; i < fields.size (); ++i)
  {
    if (fields[i].name == "x") fx = (int) i; else if (fields[i].name == "y") fy = (int) i; else if (fields[i].name == "z") fz = (int) i;
    else if ((fields[i].name == "rgba" || fields[i].name == "rgb") && fields[i].size == 4) fc = (int) i;
  }
  // records, array-of-structures
  std::vector<unsigned char> raw (npoints * rec);
  if (data_mode == "ascii")
  {
    std::size_t i = 0;
    while (i < npoints && std::getline (f, line))
    {
      std::istringstream ls (line);
      std::vector<std::string> tok; for (std::string t; ls >> t;) tok.push_back (t);
      if (tok.empty ()) continue;
      std::size_t k = 0;
      for (auto& fd : fields)
        for (int c = 0; c < fd.count; ++c, ++k)
        {
          if (k >= tok.size ()) return "short ascii record in " + path;
          detail::token_to_bytes (tok[k], fd, raw.data () + i * rec + fd.offset + (std::size_t) c * fd.size);
        }
      ++i;
    }
    if (i != npoints) return "ascii PCD ends after " + std::to_string (i) + " of " + std::to_string (npoints) + " points";
  }
  else if (data_mode == "binary")
  {
    f.read ((char*) raw.data (), (std::streamsize) raw.size ());
    if ((std::size_t) f.gcount () != raw.size ()) return "binary PCD is truncated: " + path;
  }
  else if (data_mode == "binary_compressed")
  {
    std::uint32_t csize = 0, usize = 0;
    f.read ((char*) &csize, 4); f.read ((char*) &usize, 4);
    if (!f || usize != raw.size ()) return "binary_compressed PCD: size header does not match the fields";
    std::vector<unsigned char> comp (csize), soa (usize);
    f.read ((char*) comp.data (), csize);
    if ((std::size_t) f.gcount () != csize) return "binary_compressed PCD is truncated";
    if (usize && !lzf_decompress (comp.data (), csize, soa.data (), usize)) return "binary_compressed PCD: corrupt LZF stream";
    std::size_t base = 0;                                       // structure-of-arrays -> records
    for (auto& fd : fields)
    {
      std::size_t w = (std::size_t) fd.size * fd.count;
      for (std::size_t i = 0; i < npoints; ++i) std::memcpy (raw.data () + i * rec + fd.offset, soa.data () + base + i * w, w);
      base += w * npoints;
    }
  }
  else return "unknown DATA mode " + data_mode;
  cloud.points.resize (npoints);
  cloud.has_color = fc >= 0;
  const float nan = std::numeric_limits<float>::quiet_NaN ();
  for (std::size_t i = 0; i < npoints; ++i)
  {
    const unsigned char* r = raw.data () + i * rec;
    PointXYZRGBA16& p = cloud.points[i];
    p.x = fx >= 0 ? (float) detail::scalar_from (r + fields[fx].offset, fields[fx]) : 0.f;
    p.y = fy >= 0 ? (float) detail::scalar_from (r + fields[fy].offset, fields[fy]) : 0.f;
    p.z = fz >= 0 ? (float) detail::scalar_from (r + fields[fz].offset, fields[fz]) : 0.f;
    (void) nan;
    if (fc >= 0) { const unsigned char* c = r + fields[fc].offset; p.b = c[0]; p.g = c[1]; p.r = c[2]; p.a = c[3]; }
    else { p.b = p.g = p.r = 0; p.a = 255; }
  }
  return "";
}

// Writer (tests, tools): x y z [rgba]; mode "ascii" | "binary" | "binary_compressed".
inline std::string save_pcd (const std::string& path, const Cloud& cloud, const std::string& mode, bool with_color)
{
  std::ofstream f (path, std::ios::binary);
  if (!f) return "cannot write " + path;
  const std::size_t n = cloud.points.size ();
  std::uint32_t w = cloud.width ? cloud.width : (std::uint32_t) n, h = cloud.height ? cloud.height : 1;
  f << "# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\n";
  f << (with_color ? "FIELDS x y z rgba\nSIZE 4 4 4 4\nTYPE F F F U\nCOUNT 1 1 1 1\n" : "FIELDS x y z\nSIZE 4 4 4\nTYPE F F F\nCOUNT 1 1 1\n");
  f << "WIDTH " << w << "\nHEIGHT " << h << "\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS " << n << "\nDATA " << mode << "\n";
  const std::size_t rec = with_color ? 16 : 12;
  if (mode == "ascii")
  {
    char buf[128];
    for (auto& p : cloud.points)
    {
      auto num = [&] (float v) { if (v != v) return std::string ("nan"); std::snprintf (buf, sizeof buf, "%.9g", v); return std::string (buf); };
      f << num (p.x) << ' ' << num (p.y) << ' ' << num (p.z);
      if (with_color) { std::uint32_t c; std::memcpy (&c, &p.b, 4); f << ' ' << c; }
      f << '\n';
    }
  }
  else if (mode == "binary")
    for (auto& p : cloud.points) f.write ((const char*) &p, (std::streamsize) rec);
  else if (mode == "binary_compressed")
  {
    std::vector<unsigned char> soa (n * rec);
    for (std::size_t i = 0; i < n; ++i)
    {
      std::memcpy (&soa[i * 4], &cloud.points[i].x, 4); std::memcpy (&soa[n * 4 + i * 4], &cloud.points[i].y, 4);
      std::memcpy (&soa[n * 8 + i * 4], &cloud.points[i].z, 4);
      if (with_color) std::memcpy (&soa[n * 12 + i * 4], &cloud.points[i].b, 4);
    }
    std::vector<unsigned char> comp = lzf_store (soa.data (), soa.size ());
    std::uint32_t cs = (std::uint32_t) comp.size (), us = (std::uint32_t) soa.size ();
    f.write ((const char*) &cs, 4); f.write ((const char*) &us, 4); f.write ((const char*) comp.data (), cs);
  }
  else return "unknown DATA mode " + mode;
  return f ? "" : "write failed: " + path;
}

} // namespace b200prog
