// pfb_model_files.cu — pfb_model_from_files(): URDF + parameter YAML -> PfbModel, inside the C-ABI (host code only).
//
// Replaces what the reference's drone constructors do with `<model>.urdf` + `<model>.yaml`:
//   p.loadURDF(..., flags=URDF_USE_INERTIA_FROM_FILE)          core/abstractions/base_drone.py:104-122
//   QuadX.__init__      motor / drag / PID tables               core/drones/quadx.py:84-197
//   Fixedwing.__init__  5 lifting surfaces + motor              core/drones/fixedwing.py:70-166
//   Rocket.__init__     finlets + booster + gimbal + body drag  core/drones/rocket.py:82-208
//   LiftingSurface.__init__ host precomputation                 core/abstractions/lifting_surfaces.py:180-264
// The Python mirror of this function is pyflyt_b200/models/{urdf,tables}.py; tests/test_model_files.py checks that both
// produce the same table field by field.  Only what those files need is parsed: a URDF with fixed joints (elements,
// attributes, comments; the text after the first </robot> is ignored — rocket.urdf carries a stray second one) and a YAML
// subset (nested block mappings, scalars, flow sequences of numbers, comments).
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <string>
#include <vector>

#include "../../include/pyflyt_b200.h"
#include "pfb_context.h"

namespace {

// ---------------------------------------------------------------------------------------------------
// small linear algebra (double, row-major 3x3)
// ---------------------------------------------------------------------------------------------------
struct V3 { double x, y, z; };
struct M3 { double m[9]; };
inline V3 operator+(V3 a, V3 b) { return V3{a.x + b.x, a.y + b.y, a.z + b.z}; }
inline V3 operator-(V3 a, V3 b) { return V3{a.x - b.x, a.y - b.y, a.z - b.z}; }
inline V3 operator*(double s, V3 a) { return V3{s * a.x, s * a.y, s * a.z}; }
inline double dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
inline V3 cross(V3 a, V3 b) { return V3{a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
inline M3 eye() { return M3{{1, 0, 0, 0, 1, 0, 0, 0, 1}}; }
inline M3 zero3() { return M3{{0, 0, 0, 0, 0, 0, 0, 0, 0}}; }
inline M3 mul(const M3& a, const M3& b) {
  M3 c = zero3();
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j)
      for (int k = 0; k < 3; ++k) c.m[3 * i + j] += a.m[3 * i + k] * b.m[3 * k + j];
  return c;
}
inline M3 transpose(const M3& a) { return M3{{a.m[0], a.m[3], a.m[6], a.m[1], a.m[4], a.m[7], a.m[2], a.m[5], a.m[8]}}; }
inline V3 mul(const M3& a, V3 v) {
  return V3{a.m[0] * v.x + a.m[1] * v.y + a.m[2] * v.z, a.m[3] * v.x + a.m[4] * v.y + a.m[5] * v.z, a.m[6] * v.x + a.m[7] * v.y + a.m[8] * v.z};
}
// URDF fixed-axis roll-pitch-yaw -> Rz(yaw) Ry(pitch) Rx(roll)
inline M3 rpy_to_matrix(V3 rpy) {
  const double cr = cos(rpy.x), sr = sin(rpy.x), cp = cos(rpy.y), sp = sin(rpy.y), cy = cos(rpy.z), sy = sin(rpy.z);
  return M3{{cy * cp, cy * sp * sr - sy * cr, cy * sp * cr + sy * sr, sy * cp, sy * sp * sr + cy * cr, sy * sp * cr - cy * sr, -sp, cp * sr, cp * cr}};
}

// ---------------------------------------------------------------------------------------------------
// XML (the subset a URDF uses)
// ---------------------------------------------------------------------------------------------------
struct XmlNode {
  std::string name;
  std::map<std::string, std::string> attr;
  std::vector<XmlNode> kids;
  const XmlNode* child(const char* n) const {
    for (const XmlNode& k : kids)
      if (k.name == n) return &k;
    return nullptr;
  }
  const char* get(const char* a) const {
    auto it = attr.find(a);
    return it == attr.end() ? nullptr : it->second.c_str();
  }
};

struct XmlParser {
  const std::string& s;
  size_t i = 0;
  std::string err;
  explicit XmlParser(const std::string& text) : s(text) {}
  void skip_ws() { while (i < s.size() && isspace((unsigned char)s[i])) ++i; }
  bool starts(const char* lit) const { return s.compare(i, strlen(lit), lit) == 0; }
  // skips whitespace, text, comments, processing instructions and doctype declarations up to the next tag
  bool skip_misc() {
    for (;;) {
      while (i < s.size() && s[i] != '<') ++i;  // character data is not used by URDF
      if (i >= s.size()) return true;
      if (starts("<!--")) {
        size_t e = s.find("-->", i + 4);
        if (e == std::string::npos) { err = "unterminated comment"; return false; }
        i = e + 3;
      } else if (starts("<?")) {
        size_t e = s.find("?>", i + 2);
        if (e == std::string::npos) { err = "unterminated processing instruction"; return false; }
        i = e + 2;
      } else if (starts("<!")) {
        size_t e = s.find('>', i);
        if (e == std::string::npos) { err = "unterminated declaration"; return false; }
        i = e + 1;
      } else {
        return true;
      }
    }
  }
  static bool name_char(char c) { return isalnum((unsigned char)c) || c == '_' || c == '-' || c == ':' || c == '.'; }
  bool parse_element(XmlNode& out) {
    if (!skip_misc()) return false;
    if (i >= s.size() || s[i] != '<' || (i + 1 < s.size() && s[i + 1] == '/')) { err = "expected an element"; return false; }
    ++i;
    size_t b = i;
    while (i < s.size() && name_char(s[i])) ++i;
    out.name = s.substr(b, i - b);
    if (out.name.empty()) { err = "empty element name"; return false; }
    for (;;) {
      skip_ws();
      if (i >= s.size()) { err = "unterminated tag <" + out.name + ">"; return false; }
      if (s[i] == '/') {
        if (i + 1 >= s.size() || s[i + 1] != '>') { err = "malformed tag <" + out.name + ">"; return false; }
        i += 2;
        return true;
      }
      if (s[i] == '>') { ++i; break; }
      b = i;
      while (i < s.size() && name_char(s[i])) ++i;
      std::string key = s.substr(b, i - b);
      skip_ws();
      if (key.empty() || i >= s.size() || s[i] != '=') { err = "malformed attribute in <" + out.name + ">"; return false; }
      ++i;
      skip_ws();
      if (i >= s.size() || (s[i] != '"' && s[i] != '\'')) { err = "unquoted attribute value in <" + out.name + ">"; return false; }
      const char q = s[i++];
      b = i;
      while (i < s.size() && s[i] != q) ++i;
      if (i >= s.size()) { err = "unterminated attribute value in <" + out.name + ">"; return false; }
      out.attr[key] = s.substr(b, i - b);
      ++i;
    }
    for (;;) {  // children until the matching end tag
      if (!skip_misc()) return false;
      if (i >= s.size()) { err = "missing </" + out.name + ">"; return false; }
      if (s[i + 1] == '/') {
        size_t e = s.find('>', i);
        if (e == std::string::npos) { err = "unterminated end tag"; return false; }
        std::string n = s.substr(i + 2, e - i - 2);
        while (!n.empty() && isspace((unsigned char)n.back())) n.pop_back();
        if (n != out.name) { err = "</" + n + "> closes <" + out.name + ">"; return false; }
        i = e + 1;
        return true;
      }
      XmlNode k;
      if (!parse_element(k)) return false;
      out.kids.push_back(std::move(k));
    }
  }
};

bool read_file(const char* path, std::string& out) {
  FILE* f = fopen(path, "rb");
  if (!f) return false;
  char buf[65536];
  size_t n;
  while ((n = fread(buf, 1, sizeof(buf), f)) > 0) out.append(buf, n);
  fclose(f);
  return true;
}

bool parse_doubles(const char* text, int n, double scale, double* out, bool exact) {
  for (int k = 0; k < n; ++k) out[k] = 0.0;
  if (!text) return !exact;
  const char* p = text;
  int k = 0;
  while (*p) {
    while (*p && (isspace((unsigned char)*p) || *p == ',')) ++p;
    if (!*p) break;
    char* e = nullptr;
    double v = strtod(p, &e);
    if (e == p) return false;
    if (k < n) out[k] = v * scale;
    ++k;
    p = e;
  }
  return exact ? k == n : k <= n;
}
V3 vec_attr(const XmlNode* node, const char* a, bool& ok) {
  double v[3] = {0, 0, 0};
  if (node && node->get(a) && !parse_doubles(node->get(a), 3, 1.0, v, true)) ok = false;
  return V3{v[0], v[1], v[2]};
}

// ---------------------------------------------------------------------------------------------------
// link table (pyflyt_b200/models/urdf.py::load_urdf_links)
// ---------------------------------------------------------------------------------------------------
struct Shape { int kind; double dims[3]; V3 at; M3 rot; };
struct Link {
  int index;  // -1 = base, i = i-th <joint> in file order (what PyBullet numbers the child link)
  std::string name;
  double mass;
  V3 com;      // inertial-frame origin in the base inertial frame
  M3 inertia;  // about the link COM, base-frame axes
  std::vector<Shape> shapes;
};

struct Inertial { V3 xyz, rpy; double mass; M3 tensor; };
bool inertial_of(const XmlNode& link, Inertial& o) {
  o = Inertial{V3{0, 0, 0}, V3{0, 0, 0}, 0.0, zero3()};
  const XmlNode* ine = link.child("inertial");
  if (!ine) return true;
  bool ok = true;
  const XmlNode* org = ine->child("origin");
  o.xyz = vec_attr(org, "xyz", ok);
  o.rpy = vec_attr(org, "rpy", ok);
  if (const XmlNode* m = ine->child("mass")) o.mass = m->get("value") ? atof(m->get("value")) : 0.0;
  if (const XmlNode* it = ine->child("inertia")) {
    auto g = [&](const char* k) { return it->get(k) ? atof(it->get(k)) : 0.0; };
    const double ixx = g("ixx"), ixy = g("ixy"), ixz = g("ixz"), iyy = g("iyy"), iyz = g("iyz"), izz = g("izz");
    o.tensor = M3{{ixx, ixy, ixz, ixy, iyy, iyz, ixz, iyz, izz}};
  }
  return ok;
}

// link_frame: the primitives and inertial frames in the base LINK frame (static bodies, which loadURDF places by that frame),
// and every geometry must be a box, a cylinder or a sphere; else in the base inertial frame, meshes and planes skipped
int load_urdf_links(const char* path, std::vector<Link>& links, bool link_frame = false) {
  std::string text;
  if (!read_file(path, text)) return fail("cannot read URDF %s", path);
  size_t cut = text.find("</robot>");
  if (cut != std::string::npos) text.resize(cut + 8);
  XmlParser xp(text);
  XmlNode robot;
  if (!xp.parse_element(robot)) return fail("%s: XML error near byte %zu: %s", path, xp.i, xp.err.c_str());
  if (robot.name != "robot") return fail("%s: root element is <%s>, expected <robot>", path, robot.name.c_str());

  std::map<std::string, const XmlNode*> link_nodes;
  std::vector<std::string> link_order;
  struct Joint { std::string parent, child; V3 xyz, rpy; };
  std::vector<Joint> joints;
  for (const XmlNode& k : robot.kids) {
    if (k.name == "link") {
      const char* n = k.get("name");
      if (!n) return fail("%s: <link> without a name", path);
      link_nodes[n] = &k;
      link_order.push_back(n);
    } else if (k.name == "joint") {
      const char* type = k.get("type");
      if (!type || strcmp(type, "fixed") != 0)
        return fail("%s: joint '%s' is '%s'; the batched stepper models a single free rigid body, so every joint must be 'fixed'", path,
                    k.get("name") ? k.get("name") : "?", type ? type : "?");
      const XmlNode *p = k.child("parent"), *c = k.child("child");
      if (!p || !c || !p->get("link") || !c->get("link")) return fail("%s: joint '%s' lacks parent / child", path, k.get("name") ? k.get("name") : "?");
      bool ok = true;
      Joint j{p->get("link"), c->get("link"), vec_attr(k.child("origin"), "xyz", ok), vec_attr(k.child("origin"), "rpy", ok)};
      if (!ok) return fail("%s: malformed origin in joint '%s'", path, k.get("name") ? k.get("name") : "?");
      joints.push_back(j);
    }
  }
  // root = the link that is nobody's child
  std::string base;
  int n_roots = 0;
  for (const std::string& n : link_order) {
    bool is_child = false;
    for (const Joint& j : joints) is_child = is_child || j.child == n;
    if (!is_child) { base = n; ++n_roots; }
  }
  if (n_roots != 1) return fail("%s: expected one root link, found %d", path, n_roots);
  for (const Joint& j : joints)
    if (!link_nodes.count(j.parent) || !link_nodes.count(j.child)) return fail("%s: joint refers to an unknown link", path);

  // URDF link frames relative to the base link frame
  struct Pose { V3 t; M3 r; };
  std::map<std::string, Pose> pose;
  pose[base] = Pose{V3{0, 0, 0}, eye()};
  std::vector<Joint> todo = joints;
  while (!todo.empty()) {
    std::vector<Joint> rest;
    for (const Joint& j : todo) {
      auto it = pose.find(j.parent);
      if (it != pose.end()) pose[j.child] = Pose{it->second.t + mul(it->second.r, j.xyz), mul(it->second.r, rpy_to_matrix(j.rpy))};
      else rest.push_back(j);
    }
    if (rest.size() == todo.size()) return fail("%s: joint tree is disconnected", path);
    todo.swap(rest);
  }

  Inertial bi;
  if (!inertial_of(*link_nodes[base], bi)) return fail("%s: malformed inertial origin in link '%s'", path, base.c_str());
  if (link_frame) {  // a static body: its base inertial frame may be offset (pfb_set_static_pose places it), not rotated
    if (bi.rpy.x != 0.0 || bi.rpy.y != 0.0 || bi.rpy.z != 0.0)
      return fail("%s: the inertial frame of base link '%s' is rotated; a static body's may only be offset", path, base.c_str());
    bi.xyz = V3{0, 0, 0};
  }
  const M3 base_rot_t = transpose(rpy_to_matrix(bi.rpy));
  auto rebase_t = [&](V3 t) { return mul(base_rot_t, t - bi.xyz); };
  auto rebase_r = [&](const M3& r) { return mul(base_rot_t, r); };

  std::vector<std::string> names;
  names.push_back(base);
  for (const Joint& j : joints) names.push_back(j.child);
  links.clear();
  for (size_t idx = 0; idx < names.size(); ++idx) {
    const XmlNode& node = *link_nodes[names[idx]];
    const Pose& f = pose[names[idx]];
    Inertial in;
    if (!inertial_of(node, in)) return fail("%s: malformed inertial origin in link '%s'", path, names[idx].c_str());
    Link lk;
    lk.index = (int)idx - 1;
    lk.name = names[idx];
    lk.mass = in.mass;
    lk.com = rebase_t(f.t + mul(f.r, in.xyz));
    const M3 axes = rebase_r(mul(f.r, rpy_to_matrix(in.rpy)));
    lk.inertia = mul(mul(axes, in.tensor), transpose(axes));
    for (const XmlNode& col : node.kids) {
      if (col.name != "collision") continue;
      bool ok = true;
      const XmlNode* org = col.child("origin");
      const V3 cxyz = vec_attr(org, "xyz", ok), crpy = vec_attr(org, "rpy", ok);
      if (!ok) return fail("%s: malformed collision origin in link '%s'", path, names[idx].c_str());
      const XmlNode* geo = col.child("geometry");
      if (!geo) continue;
      Shape sh;
      sh.at = rebase_t(f.t + mul(f.r, cxyz));
      sh.rot = rebase_r(mul(f.r, rpy_to_matrix(crpy)));
      sh.dims[0] = sh.dims[1] = sh.dims[2] = 0.0;
      if (const XmlNode* b = geo->child("box")) {
        sh.kind = PFB_SHAPE_BOX;
        if (!parse_doubles(b->get("size"), 3, 1.0, sh.dims, true)) return fail("%s: malformed box size in link '%s'", path, names[idx].c_str());
      } else if (const XmlNode* c = geo->child("cylinder")) {
        sh.kind = PFB_SHAPE_CYLINDER;
        sh.dims[0] = c->get("radius") ? atof(c->get("radius")) : 0.0;
        sh.dims[1] = c->get("length") ? atof(c->get("length")) : 0.0;
      } else if (const XmlNode* s = geo->child("sphere")) {
        sh.kind = PFB_SHAPE_SPHERE;
        sh.dims[0] = s->get("radius") ? atof(s->get("radius")) : 0.0;
      } else if (link_frame) {
        return fail("%s: link '%s' has a collision geometry other than a box, a cylinder or a sphere; static bodies are boxes and cylinders", path,
                    names[idx].c_str());
      } else {
        continue;  // meshes / planes carry no analytic ground test
      }
      lk.shapes.push_back(sh);
    }
    links.push_back(std::move(lk));
  }
  return 0;
}

// composite rigid body about the base origin, base axes (urdf.py::composite_rigid_body); skip = link index whose mass and
// inertia are taken as zero (the rocket's fuel tank: boosters.py:207-212), -2 = none
void composite(const std::vector<Link>& links, int skip, double& M, V3& first, M3& I_O) {
  M = 0.0;
  first = V3{0, 0, 0};
  I_O = zero3();
  for (const Link& lk : links) {
    const bool off = lk.index == skip;
    const double m = off ? 0.0 : lk.mass;
    const V3 r = lk.com;
    M += m;
    first = first + m * r;
    const double rr = dot(r, r);
    const double rv[3] = {r.x, r.y, r.z};
    for (int a = 0; a < 3; ++a)
      for (int b = 0; b < 3; ++b) I_O.m[3 * a + b] += (off ? 0.0 : lk.inertia.m[3 * a + b]) + m * ((a == b ? rr : 0.0) - rv[a] * rv[b]);
  }
}

// ---------------------------------------------------------------------------------------------------
// YAML subset: nested block mappings -> "a.b.c" keys; values: scalar text or a flow sequence of numbers
// ---------------------------------------------------------------------------------------------------
struct Yaml {
  std::map<std::string, std::string> scalar;
  std::map<std::string, std::vector<double>> list;
  bool has(const std::string& k) const { return scalar.count(k) || list.count(k); }
};

std::string strip(const std::string& s) {
  size_t b = 0, e = s.size();
  while (b < e && isspace((unsigned char)s[b])) ++b;
  while (e > b && isspace((unsigned char)s[e - 1])) --e;
  return s.substr(b, e - b);
}
// removes a trailing comment that is not inside quotes
std::string strip_comment(const std::string& s) {
  char q = 0;
  for (size_t i = 0; i < s.size(); ++i) {
    const char c = s[i];
    if (q) { if (c == q) q = 0; }
    else if (c == '"' || c == '\'') q = c;
    else if (c == '#' && (i == 0 || isspace((unsigned char)s[i - 1]))) return s.substr(0, i);
  }
  return s;
}

int load_yaml(const char* path, Yaml& y) {
  std::string text;
  if (!read_file(path, text)) return fail("cannot read parameter file %s", path);
  std::vector<std::pair<int, std::string>> stack;  // (indent, key) of the open mappings
  size_t pos = 0;
  int lineno = 0;
  while (pos <= text.size()) {
    size_t e = text.find('\n', pos);
    if (e == std::string::npos) e = text.size();
    std::string raw = text.substr(pos, e - pos);
    pos = e + 1;
    ++lineno;
    if (!raw.empty() && raw.back() == '\r') raw.pop_back();
    std::string line = strip_comment(raw);
    if (strip(line).empty()) { if (e == text.size()) break; continue; }
    if (strip(line) == "---") continue;
    int indent = 0;
    while (indent < (int)line.size() && line[indent] == ' ') ++indent;
    if (indent < (int)line.size() && line[indent] == '\t') return fail("%s:%d: tabs are not valid YAML indentation", path, lineno);
    size_t colon = std::string::npos;
    {
      char q = 0;
      for (size_t i = indent; i < line.size(); ++i) {
        const char c = line[i];
        if (q) { if (c == q) q = 0; }
        else if (c == '"' || c == '\'') q = c;
        else if (c == ':' && (i + 1 == line.size() || isspace((unsigned char)line[i + 1]))) { colon = i; break; }
      }
    }
    if (colon == std::string::npos) return fail("%s:%d: expected `key: value`", path, lineno);
    const std::string key = strip(line.substr(indent, colon - indent));
    std::string val = strip(line.substr(colon + 1));
    while (!stack.empty() && stack.back().first >= indent) stack.pop_back();
    std::string full;
    for (auto& s : stack) full += s.second + ".";
    full += key;
    if (val.empty()) {
      stack.push_back({indent, key});
    } else if (val[0] == '[') {
      while (val.find(']') == std::string::npos && pos <= text.size()) {  // a flow sequence continued on the next lines
        size_t e2 = text.find('\n', pos);
        if (e2 == std::string::npos) e2 = text.size();
        val += " " + strip(strip_comment(text.substr(pos, e2 - pos)));
        pos = e2 + 1;
        ++lineno;
      }
      const size_t close = val.find(']');
      if (close == std::string::npos) return fail("%s:%d: unterminated flow sequence", path, lineno);
      std::vector<double> v;
      const std::string body = val.substr(1, close - 1);
      const char* p = body.c_str();
      while (*p) {
        while (*p && (isspace((unsigned char)*p) || *p == ',')) ++p;
        if (!*p) break;
        char* end = nullptr;
        const double d = strtod(p, &end);
        if (end == p) return fail("%s:%d: non-numeric entry in the sequence of `%s`", path, lineno, full.c_str());
        v.push_back(d);
        p = end;
      }
      y.list[full] = v;
    } else {
      if (val.size() >= 2 && (val[0] == '"' || val[0] == '\'') && val.back() == val[0]) val = val.substr(1, val.size() - 2);
      y.scalar[full] = val;
    }
    if (e == text.size()) break;
  }
  return 0;
}

// numeric scalar (YAML 1.1 core: decimal / exponent floats with an optional sign, `_` separators not used by the reference)
int yaml_num(const Yaml& y, const char* path, const std::string& key, double& out) {
  auto it = y.scalar.find(key);
  if (it == y.scalar.end()) return fail("%s: missing parameter `%s`", path, key.c_str());
  const char* p = it->second.c_str();
  char* e = nullptr;
  out = strtod(p, &e);
  if (e == p || *e != 0) return fail("%s: parameter `%s` is not a number: '%s'", path, key.c_str(), p);
  return 0;
}
int yaml_bool(const Yaml& y, const char* path, const std::string& key, int& out) {
  auto it = y.scalar.find(key);
  if (it == y.scalar.end()) return fail("%s: missing parameter `%s`", path, key.c_str());
  std::string v = it->second;
  for (char& c : v) c = (char)tolower((unsigned char)c);
  if (v == "true" || v == "yes" || v == "on") out = 1;
  else if (v == "false" || v == "no" || v == "off") out = 0;
  else return fail("%s: parameter `%s` is not a boolean: '%s'", path, key.c_str(), it->second.c_str());
  return 0;
}
// scalar or list of up to 3 numbers, zero padded (PID gains: kp: [a, b, c] | kp: a)
int yaml_vec3(const Yaml& y, const char* path, const std::string& key, double* out) {
  out[0] = out[1] = out[2] = 0.0;
  auto it = y.list.find(key);
  if (it != y.list.end()) {
    if (it->second.size() > 3) return fail("%s: `%s` has more than 3 entries", path, key.c_str());
    for (size_t k = 0; k < it->second.size(); ++k) out[k] = it->second[k];
    return 0;
  }
  return yaml_num(y, path, key, out[0]);
}

const Link* find_link(const std::vector<Link>& links, int index) {
  for (const Link& l : links)
    if (l.index == index) return &l;
  return nullptr;
}
void put3(double* dst, V3 v) { dst[0] = v.x; dst[1] = v.y; dst[2] = v.z; }

// lifting_surfaces.py:217-262 on the host
int fill_surface(PfbSurface& s, const Link& link, V3 lift, V3 fwd, const Yaml& y, const char* ypath, const std::string& sec, double dt) {
  lift = (1.0 / sqrt(dot(lift, lift))) * lift;
  fwd = (1.0 / sqrt(dot(fwd, fwd))) * fwd;
  double chord, span, ftc, cl2d, eta, a0, asp, asn, cd0, defl, tau;
  if (yaml_num(y, ypath, sec + ".chord", chord) || yaml_num(y, ypath, sec + ".span", span) || yaml_num(y, ypath, sec + ".flap_to_chord", ftc) ||
      yaml_num(y, ypath, sec + ".Cl_alpha_2D", cl2d) || yaml_num(y, ypath, sec + ".eta", eta) || yaml_num(y, ypath, sec + ".alpha_0_base", a0) ||
      yaml_num(y, ypath, sec + ".alpha_stall_P_base", asp) || yaml_num(y, ypath, sec + ".alpha_stall_N_base", asn) ||
      yaml_num(y, ypath, sec + ".Cd_0", cd0) || yaml_num(y, ypath, sec + ".deflection_limit", defl) || yaml_num(y, ypath, sec + ".tau", tau))
    return -1;
  const double aspect = span / chord;
  const double theta_f = acos(2.0 * ftc - 1.0);
  const double deg = M_PI / 180.0;
  put3(s.pos, link.com);
  put3(s.lift_unit, lift);
  put3(s.drag_unit, fwd);
  put3(s.torque_unit, cross(lift, fwd));
  s.Cl_alpha_3D = cl2d * (aspect / (aspect + ((2.0 * (aspect + 4.0)) / (aspect + 2.0))));
  s.aspect = aspect;
  s.flap_to_chord = ftc;
  s.aero_tau = 1.0 - ((theta_f - sin(theta_f)) / M_PI);
  s.eta = eta;
  s.alpha_0_base = a0 * deg;
  s.alpha_stall_P_base = asp * deg;
  s.alpha_stall_N_base = asn * deg;
  s.Cd_0 = cd0;
  s.deflection_limit_deg = defl;
  s.dt_over_tau = dt / tau;
  s.area = chord * span;
  s.chord = chord;
  s.half_rho = 0.5 * 1.225;
  return 0;
}

}  // namespace

extern "C" int pfb_static_shapes_from_urdf(const char* urdf_path, double global_scaling, PfbShape* out, int cap, int* n_shapes,
                                           double inertial_origin[3]) {
  if (!urdf_path || !n_shapes || !inertial_origin || (cap > 0 && !out)) return fail("pfb_static_shapes_from_urdf: null argument");
  if (!(global_scaling > 0.0)) return fail("pfb_static_shapes_from_urdf: globalScaling must be positive, got %g", global_scaling);
  std::vector<Link> links;
  if (load_urdf_links(urdf_path, links, true)) return -1;
  int n = 0;
  for (const Link& lk : links)
    for (const Shape& s : lk.shapes) {
      if (n >= cap) return fail("%s: more than %d collision primitives", urdf_path, cap);
      PfbShape& sh = out[n++];
      memset(&sh, 0, sizeof(sh));
      sh.kind = s.kind;  // half extents / radius and half length, as pfb_model_from_files
      if (s.kind == PFB_SHAPE_BOX) { for (int c = 0; c < 3; ++c) sh.dims[c] = 0.5 * s.dims[c] * global_scaling; }
      else if (s.kind == PFB_SHAPE_CYLINDER) { sh.dims[0] = s.dims[0] * global_scaling; sh.dims[1] = 0.5 * s.dims[1] * global_scaling; }
      else sh.dims[0] = s.dims[0] * global_scaling;
      put3(sh.at, global_scaling * s.at);
      memcpy(sh.rot, s.rot.m, sizeof(s.rot.m));
    }
  *n_shapes = n;
  put3(inertial_origin, global_scaling * links[0].com);  // the base link's inertial origin, in its own frame
  return 0;
}

extern "C" int pfb_model_from_files(int kind, const char* urdf_path, const char* yaml_path, double physics_hz, double control_hz, PfbModel* out) {
  if (!urdf_path || !yaml_path || !out) return fail("pfb_model_from_files: null argument");
  if (kind != PFB_KIND_QUADX && kind != PFB_KIND_FIXEDWING && kind != PFB_KIND_ROCKET) return fail("unknown vehicle kind %d", kind);
  if (physics_hz <= 0.0) physics_hz = 240.0;  // aviary.py:79
  if (control_hz <= 0.0) control_hz = 120.0;  // quadx.py:27, fixedwing.py:23, rocket.py:35
  if (fmod(physics_hz, control_hz) != 0.0)    // base_drone.py:94-97
    return fail("`physics_hz` (%g) must be multiple of `control_hz` (%g).", physics_hz, control_hz);
  std::vector<Link> links;
  if (load_urdf_links(urdf_path, links)) return -1;
  Yaml y;
  if (load_yaml(yaml_path, y)) return -1;
  const double dt = 1.0 / physics_hz;

  PfbModel& m = *out;
  memset(&m, 0, sizeof(m));
  m.abi_version = PFB_ABI_VERSION;
  m.kind = kind;
  m.physics_hz = physics_hz;
  m.control_hz = control_hz;
  m.gravity = -9.81;
  m.max_coord_velocity = 100.0;
  {  // composite body + collision primitives (tables.py::_fill_rigid)
    double M;
    V3 first;
    M3 I;
    composite(links, -2, M, first, I);
    m.mass = M;
    put3(m.com, M > 0.0 ? (1.0 / M) * first : V3{0, 0, 0});
    memcpy(m.inertia, I.m, sizeof(I.m));
    int n = 0;
    for (const Link& lk : links)
      for (const Shape& s : lk.shapes) {
        if (n >= PFB_MAX_SHAPES) return fail("%s: too many collision primitives (max %d)", urdf_path, PFB_MAX_SHAPES);
        PfbShape& sh = m.shapes[n++];
        sh.kind = s.kind;
        if (s.kind == PFB_SHAPE_BOX) { sh.dims[0] = 0.5 * s.dims[0]; sh.dims[1] = 0.5 * s.dims[1]; sh.dims[2] = 0.5 * s.dims[2]; }
        else if (s.kind == PFB_SHAPE_CYLINDER) { sh.dims[0] = s.dims[0]; sh.dims[1] = 0.5 * s.dims[1]; sh.dims[2] = 0.0; }
        else { sh.dims[0] = s.dims[0]; sh.dims[1] = sh.dims[2] = 0.0; }
        put3(sh.at, s.at);
        memcpy(sh.rot, s.rot.m, sizeof(s.rot.m));
      }
    m.n_shapes = n;
    m.contact_factor = 0.02;
  }
  auto need_link = [&](int index, const Link*& lk) -> int {
    lk = find_link(links, index);
    return lk ? 0 : fail("%s: vehicle has no link %d", urdf_path, index);
  };

  if (kind == PFB_KIND_QUADX) {
    double total_thrust, thrust_coef, torque_coef, noise_ratio, tau, cd, area, pqr;
    if (yaml_num(y, yaml_path, "motor_params.total_thrust", total_thrust) || yaml_num(y, yaml_path, "motor_params.thrust_coef", thrust_coef) ||
        yaml_num(y, yaml_path, "motor_params.torque_coef", torque_coef) || yaml_num(y, yaml_path, "motor_params.noise_ratio", noise_ratio) ||
        yaml_num(y, yaml_path, "motor_params.tau", tau) || yaml_num(y, yaml_path, "drag_params.drag_coef_xyz", cd) ||
        yaml_num(y, yaml_path, "drag_params.drag_area_xyz", area) || yaml_num(y, yaml_path, "drag_params.drag_coef_pqr", pqr))
      return -1;
    m.n_motors = 4;
    const double max_rpm = sqrt(total_thrust / (4.0 * thrust_coef));                   // quadx.py:111-113
    const double tq[4] = {-torque_coef, -torque_coef, +torque_coef, +torque_coef};     // quadx.py:94-101
    for (int i = 0; i < 4; ++i) {
      const Link* lk;
      if (need_link(i, lk)) return -1;
      put3(m.motor_pos[i], lk->com);
      m.motor_axis[i][2] = 1.0;
      m.thrust_coef[i] = thrust_coef;
      m.torque_coef[i] = tq[i];
      m.max_rpm[i] = max_rpm;
      m.motor_dt_over_tau[i] = dt / tau;
      m.motor_noise_ratio[i] = noise_ratio;
    }
    const Link* body;
    if (need_link(4, body)) return -1;  // body_ids = [4], quadx.py:148
    m.n_bodies = 1;
    put3(m.body_pos, body->com);
    const double k = 0.5 * 1.225 * cd * area;  // boring_bodies.py:63
    m.drag_const[0] = m.drag_const[1] = m.drag_const[2] = k;
    m.drag_coef_pqr = pqr;
    const char* names[6] = {"ang_vel", "ang_pos", "lin_vel", "lin_pos", "z_vel", "z_pos"};
    const char* gains[4] = {"kp", "ki", "kd", "lim"};
    for (int p = 0; p < 6; ++p)
      for (int g = 0; g < 4; ++g)
        if (yaml_vec3(y, yaml_path, std::string("control_params.") + names[p] + "." + gains[g], m.pid[p][g])) return -1;
    const double mm[4][4] = {{-1, -1, -1, +1}, {+1, +1, -1, +1}, {+1, -1, +1, +1}, {-1, +1, +1, +1}};  // quadx.py:130-137
    memcpy(m.motor_map, mm, sizeof(mm));
  } else if (kind == PFB_KIND_FIXEDWING) {
    double total_thrust, thrust_coef, torque_coef, noise_ratio, tau;
    if (yaml_num(y, yaml_path, "motor_params.total_thrust", total_thrust) || yaml_num(y, yaml_path, "motor_params.thrust_coef", thrust_coef) ||
        yaml_num(y, yaml_path, "motor_params.torque_coef", torque_coef) || yaml_num(y, yaml_path, "motor_params.noise_ratio", noise_ratio) ||
        yaml_num(y, yaml_path, "motor_params.tau", tau))
      return -1;
    const Link* ml;
    if (need_link(0, ml)) return -1;
    m.n_motors = 1;
    put3(m.motor_pos[0], ml->com);
    m.motor_axis[0][0] = 1.0;
    m.thrust_coef[0] = thrust_coef;
    m.torque_coef[0] = torque_coef;
    m.max_rpm[0] = sqrt(total_thrust / thrust_coef);  // fixedwing.py:149-151
    m.motor_dt_over_tau[0] = dt / tau;
    m.motor_noise_ratio[0] = noise_ratio;
    // order and link ids: fixedwing.py:79-138
    struct Spec { int link; V3 lift; const char* key; };
    const Spec spec[5] = {{3, V3{0, 0, 1}, "left_wing_flapped_params"}, {4, V3{0, 0, 1}, "right_wing_flapped_params"},
                          {1, V3{0, 0, 1}, "horizontal_tail_params"},   {2, V3{0, 1, 0}, "vertical_tail_params"},
                          {5, V3{0, 0, 1}, "main_wing_params"}};
    m.n_surfaces = 5;
    for (int s = 0; s < 5; ++s) {
      const Link* lk;
      if (need_link(spec[s].link, lk)) return -1;
      if (fill_surface(m.surfaces[s], *lk, spec[s].lift, V3{1, 0, 0}, y, yaml_path, spec[s].key, dt)) return -1;
    }
    m.starting_velocity[0] = 20.0;  // fixedwing.py:35
  } else {
    double cdx, cdy, cdz, ax, ay, az;
    if (yaml_num(y, yaml_path, "body_params.drag_coef_x", cdx) || yaml_num(y, yaml_path, "body_params.drag_coef_y", cdy) ||
        yaml_num(y, yaml_path, "body_params.drag_coef_z", cdz) || yaml_num(y, yaml_path, "body_params.area_x", ax) ||
        yaml_num(y, yaml_path, "body_params.area_y", ay) || yaml_num(y, yaml_path, "body_params.area_z", az))
      return -1;
    const Link *tank, *booster;
    if (need_link(0, tank) || need_link(1, booster)) return -1;  // body_ids = [0] rocket.py:92, fueltank_ids = [0], booster_ids = [1] :163-164
    m.n_bodies = 1;
    put3(m.body_pos, tank->com);
    m.drag_const[0] = 0.5 * 1.225 * cdx * ax;
    m.drag_const[1] = 0.5 * 1.225 * cdy * ay;
    m.drag_const[2] = 0.5 * 1.225 * cdz * az;
    // finlets sit on link ids 0, 1 (lift +y) and 2, 3 (lift +x): rocket.py:113-144 (sic)
    m.n_surfaces = 4;
    const V3 lifts[4] = {V3{0, 1, 0}, V3{0, 1, 0}, V3{1, 0, 0}, V3{1, 0, 0}};
    for (int s = 0; s < 4; ++s) {
      const Link* lk;
      if (need_link(s, lk)) return -1;
      if (fill_surface(m.surfaces[s], *lk, lifts[s], V3{0, 0, -1}, y, yaml_path, "finlet_params", dt)) return -1;
    }
    double total_fuel, max_rate, ixx, iyy, izz, tmin, tmax, grange, btau, gtau, noise;
    int reign;
    if (yaml_num(y, yaml_path, "booster_params.total_fuel", total_fuel) || yaml_num(y, yaml_path, "booster_params.max_fuel_rate", max_rate) ||
        yaml_num(y, yaml_path, "booster_params.inertia_ixx", ixx) || yaml_num(y, yaml_path, "booster_params.inertia_iyy", iyy) ||
        yaml_num(y, yaml_path, "booster_params.inertia_izz", izz) || yaml_num(y, yaml_path, "booster_params.min_thrust", tmin) ||
        yaml_num(y, yaml_path, "booster_params.max_thrust", tmax) || yaml_bool(y, yaml_path, "booster_params.reignitable", reign) ||
        yaml_num(y, yaml_path, "booster_params.gimbal_range_degrees", grange) || yaml_num(y, yaml_path, "booster_params.booster_tau", btau) ||
        yaml_num(y, yaml_path, "booster_params.gimbal_tau", gtau) || yaml_num(y, yaml_path, "booster_params.noise_ratio", noise))
      return -1;
    m.has_booster = 1;
    m.reignitable = reign;
    put3(m.booster_pos, booster->com);
    m.booster_axis[2] = 1.0;
    m.booster_dt_over_tau = dt / btau;
    m.booster_noise_ratio = noise;
    m.booster_min_thrust = tmin;
    m.booster_max_thrust = tmax;
    m.fuel_total_mass = total_fuel;
    m.fuel_max_rate = max_rate;
    m.fuel_max_inertia[0] = ixx; m.fuel_max_inertia[1] = iyy; m.fuel_max_inertia[2] = izz;
    put3(m.fuel_pos, tank->com);
    double Md;
    V3 firstd;
    M3 Id;
    composite(links, 0, Md, firstd, Id);  // without the tank: its mass and inertia follow the fuel level (boosters.py:207-212)
    m.dry_mass = Md;
    put3(m.dry_first_moment, firstd);
    memcpy(m.dry_inertia, Id.m, sizeof(Id.m));
    m.gimbal_unit1[0] = 1.0;
    m.gimbal_unit2[1] = 1.0;
    m.gimbal_dt_over_tau = dt / gtau;
    m.gimbal_range_rad[0] = m.gimbal_range_rad[1] = grange * (M_PI / 180.0);
    m.starting_fuel_ratio = 0.05;  // rocket.py:47 default; the caller overwrites it like `drone_options`
  }
  return 0;
}
