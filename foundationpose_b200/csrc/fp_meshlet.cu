// fp_meshlet.cu — host-side mesh preparation for the tiled crop producer (init time, fp_set_mesh):
//   * packs the vertex attributes of Utils.py:104-130 make_mesh_tensors into 16-byte records;
//   * decides whether back faces can be culled: the mesh must be CLOSED and CONSISTENTLY ORIENTED (every directed edge
//     of the position-welded mesh occurs exactly once and its reverse exactly once); the sign of the enclosed volume
//     tells which screen-space winding is front-facing.  nvdiffrast (Utils.py:182) renders both sides, so an open mesh
//     keeps both sides here too;
//   * builds meshlets by region growing over the face adjacency (nearest-centroid, normal-coherent growth from a seed
//     face): connected, compact patches of <= 64 triangles / <= 64 unique vertices, each with a bounding sphere and a
//     normal cone.
// Pure host code (no kernels); compiled with the rest of the library.
#include <math.h>
#include <stdint.h>

#include <algorithm>
#include <numeric>
#include <unordered_map>

#include "fp_common.cuh"
#include "fp_crop.cuh"

namespace fp {

namespace {

struct V3 {
  double x, y, z;
};
inline V3 sub(V3 a, V3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
inline V3 cross(V3 a, V3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
inline double dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
inline double norm(V3 a) { return sqrt(dot(a, a)); }

inline uint32_t part1by2(uint32_t x) {  // spread the low 10 bits
  x &= 0x3ff;
  x = (x | (x << 16)) & 0x30000ff;
  x = (x | (x << 8)) & 0x300f00f;
  x = (x | (x << 4)) & 0x30c30c3;
  x = (x | (x << 2)) & 0x9249249;
  return x;
}

struct PosKey {
  uint32_t a, b, c;
  bool operator==(const PosKey& o) const { return a == o.a && b == o.b && c == o.c; }
};
struct PosHash {
  size_t operator()(const PosKey& k) const {
    uint64_t h = 1469598103934665603ull;
    for (uint32_t w : {k.a, k.b, k.c}) {
      h ^= w;
      h *= 1099511628211ull;
    }
    return (size_t)h;
  }
};

}  // namespace

int build_mesh_host(int V, int F, const float* pos, const float* nrm, const float* att, int n_att, const int* faces,
                    MeshHost& out) {
  out.vpos.resize(V);
  out.vnrm.resize(V);
  out.vatt.resize(V);
  for (int v = 0; v < V; ++v) {
    out.vpos[v] = make_float4(pos[3 * v], pos[3 * v + 1], pos[3 * v + 2], 0.f);
    out.vnrm[v] = nrm ? make_float4(nrm[3 * v], nrm[3 * v + 1], nrm[3 * v + 2], 0.f) : make_float4(0.f, 0.f, 0.f, 0.f);
    out.vatt[v] = !att ? make_float4(0.f, 0.f, 0.f, 0.f)
                       : n_att == 2 ? make_float4(att[2 * v], att[2 * v + 1], 0.f, 0.f)
                                    : make_float4(att[3 * v], att[3 * v + 1], att[3 * v + 2], 0.f);
  }
  out.faces.resize(F);
  for (int f = 0; f < F; ++f) out.faces[f] = make_int4(faces[3 * f], faces[3 * f + 1], faces[3 * f + 2], 0);

  auto P = [&](int v) { return V3{pos[3 * v], pos[3 * v + 1], pos[3 * v + 2]}; };

  // ---- closedness / orientation on the position-welded mesh (texture seams duplicate vertices)
  std::vector<int> canon(V);
  {
    std::unordered_map<PosKey, int, PosHash> seen;
    seen.reserve((size_t)V * 2);
    for (int v = 0; v < V; ++v) {
      float q[3] = {pos[3 * v] + 0.f, pos[3 * v + 1] + 0.f, pos[3 * v + 2] + 0.f};  // +0 folds -0 into +0
      PosKey k;
      memcpy(&k.a, q, 4);
      memcpy(&k.b, q + 1, 4);
      memcpy(&k.c, q + 2, 4);
      auto it = seen.find(k);
      if (it == seen.end()) {
        seen.emplace(k, v);
        canon[v] = v;
      } else {
        canon[v] = it->second;
      }
    }
  }
  bool closed = true;
  {
    std::unordered_map<uint64_t, int> edges;  // directed edge (a, b) -> count
    edges.reserve((size_t)F * 4);
    for (int f = 0; f < F && closed; ++f) {
      const int i[3] = {canon[faces[3 * f]], canon[faces[3 * f + 1]], canon[faces[3 * f + 2]]};
      if (i[0] == i[1] || i[1] == i[2] || i[0] == i[2]) continue;  // degenerate after welding: covers nothing
      for (int e = 0; e < 3; ++e) {
        const uint64_t key = ((uint64_t)(uint32_t)i[e] << 32) | (uint32_t)i[(e + 1) % 3];
        if (++edges[key] > 1) closed = false;  // an edge used twice in the same direction: inconsistent winding
      }
    }
    if (closed)
      for (auto& kv : edges) {
        const uint64_t rev = (kv.first << 32) | (kv.first >> 32);
        auto it = edges.find(rev);
        if (it == edges.end() || it->second != 1) {
          closed = false;
          break;
        }
      }
  }
  double vol6 = 0.0;
  for (int f = 0; f < F; ++f) vol6 += dot(P(faces[3 * f]), cross(P(faces[3 * f + 1]), P(faces[3 * f + 2])));
  out.closed = closed ? 1 : 0;
  // camera looks down +z with x right / y down (OpenCV): a triangle whose outward normal faces the camera has a
  // NEGATIVE signed screen area (x1-x0)(y2-y0) - (y1-y0)(x2-x0); inside-out meshes (negative volume) flip that
  out.front_sign = !closed || vol6 == 0.0 ? 0 : (vol6 > 0.0 ? -1 : 1);

  // ---- face centroids / unit normals, Morton order of the centroids (seed order for disconnected pieces)
  V3 lo = {1e300, 1e300, 1e300}, hi = {-1e300, -1e300, -1e300};
  for (int v = 0; v < V; ++v) {
    const V3 p = P(v);
    lo = {std::min(lo.x, p.x), std::min(lo.y, p.y), std::min(lo.z, p.z)};
    hi = {std::max(hi.x, p.x), std::max(hi.y, p.y), std::max(hi.z, p.z)};
  }
  const double ext = std::max({hi.x - lo.x, hi.y - lo.y, hi.z - lo.z, 1e-30});
  {
    const V3 c = {(lo.x + hi.x) / 2, (lo.y + hi.y) / 2, (lo.z + hi.z) / 2};
    double r = 0;
    for (int v = 0; v < V; ++v) r = std::max(r, norm(sub(P(v), c)));
    out.bs[0] = (float)c.x;
    out.bs[1] = (float)c.y;
    out.bs[2] = (float)c.z;
    out.bs[3] = (float)(r * 1.0001 + 1e-9);
  }
  std::vector<V3> fn(F), fc(F);
  std::vector<uint64_t> key(F);
  for (int f = 0; f < F; ++f) {
    const V3 a = P(faces[3 * f]), b = P(faces[3 * f + 1]), c = P(faces[3 * f + 2]);
    V3 n = cross(sub(b, a), sub(c, a));
    const double l = norm(n);
    fn[f] = l > 0 ? V3{n.x / l, n.y / l, n.z / l} : V3{0, 0, 0};
    fc[f] = {(a.x + b.x + c.x) / 3, (a.y + b.y + c.y) / 3, (a.z + b.z + c.z) / 3};
    const uint32_t qx = (uint32_t)std::min(1023.0, (fc[f].x - lo.x) / ext * 1023.0);
    const uint32_t qy = (uint32_t)std::min(1023.0, (fc[f].y - lo.y) / ext * 1023.0);
    const uint32_t qz = (uint32_t)std::min(1023.0, (fc[f].z - lo.z) / ext * 1023.0);
    key[f] = part1by2(qx) | (part1by2(qy) << 1) | (part1by2(qz) << 2);
  }
  std::vector<int> order(F);
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return key[a] < key[b]; });

  // ---- face adjacency over the welded edges (CSR); non-manifold edges link all their faces
  std::vector<int> adj_off(F + 1, 0), adj;
  {
    std::vector<std::pair<uint64_t, int>> ef;
    ef.reserve((size_t)F * 3);
    for (int f = 0; f < F; ++f) {
      const int i[3] = {canon[faces[3 * f]], canon[faces[3 * f + 1]], canon[faces[3 * f + 2]]};
      for (int e = 0; e < 3; ++e) {
        const int a = i[e], b = i[(e + 1) % 3];
        if (a == b) continue;
        ef.push_back({((uint64_t)(uint32_t)std::min(a, b) << 32) | (uint32_t)std::max(a, b), f});
      }
    }
    std::sort(ef.begin(), ef.end());
    std::vector<std::pair<int, int>> links;
    for (size_t s0 = 0; s0 < ef.size();) {
      size_t s1 = s0;
      while (s1 < ef.size() && ef[s1].first == ef[s0].first) ++s1;
      const size_t run = std::min<size_t>(s1 - s0, 8);  // cap pathological fans
      for (size_t a = s0; a < s0 + run; ++a)
        for (size_t b = a + 1; b < s0 + run; ++b)
          if (ef[a].second != ef[b].second) {
            links.push_back({ef[a].second, ef[b].second});
            links.push_back({ef[b].second, ef[a].second});
          }
      s0 = s1;
    }
    for (auto& l : links) ++adj_off[l.first + 1];
    for (int f = 0; f < F; ++f) adj_off[f + 1] += adj_off[f];
    adj.resize(links.size());
    std::vector<int> fill(adj_off.begin(), adj_off.end() - 1);
    for (auto& l : links) adj[fill[l.first]++] = l.second;
  }

  // ---- greedy chunking
  out.meshlets.clear();
  out.ml_verts.clear();
  out.ml_tris.clear();
  std::vector<int> slot_of(V, -1);
  std::vector<int> cur_verts;
  std::vector<int> cur_faces;
  std::vector<uint2> cur_tris;
  auto flush = [&]() {
    if (cur_faces.empty()) return;
    Meshlet m;
    m.vert_off = (int)out.ml_verts.size();
    m.n_verts = (int)cur_verts.size();
    m.tri_off = (int)out.ml_tris.size();
    m.n_tris = (int)cur_faces.size();
    V3 c = {0, 0, 0};
    for (int v : cur_verts) {
      const V3 p = P(v);
      c = {c.x + p.x, c.y + p.y, c.z + p.z};
    }
    c = {c.x / m.n_verts, c.y / m.n_verts, c.z / m.n_verts};
    double r = 0;
    for (int v : cur_verts) r = std::max(r, norm(sub(P(v), c)));
    m.cx = (float)c.x;
    m.cy = (float)c.y;
    m.cz = (float)c.z;
    m.r = (float)(r * 1.0001 + 1e-9);
    V3 ax = {0, 0, 0};
    bool degenerate = false;
    for (int f : cur_faces) {
      if (dot(fn[f], fn[f]) == 0) degenerate = true;
      ax = {ax.x + fn[f].x, ax.y + fn[f].y, ax.z + fn[f].z};
    }
    const double al = norm(ax);
    m.ax = m.ay = m.az = 0.f;
    m.cutoff = -2.f;
    if (out.front_sign && !degenerate && al > 1e-9) {
      ax = {ax.x / al, ax.y / al, ax.z / al};
      double mn = 1.0;
      for (int f : cur_faces) mn = std::min(mn, dot(ax, fn[f]));
      m.ax = (float)ax.x;
      m.ay = (float)ax.y;
      m.az = (float)ax.z;
      m.cutoff = (float)mn;
    }
    for (int v : cur_verts) {
      out.ml_verts.push_back(v);
      slot_of[v] = -1;
    }
    for (const uint2& t : cur_tris) out.ml_tris.push_back(t);
    out.meshlets.push_back(m);
    cur_verts.clear();
    cur_faces.clear();
    cur_tris.clear();
  };
  // ---- region growing: a meshlet starts at a seed face and repeatedly takes, from the faces adjacent to it, the
  // one whose centroid is nearest to the meshlet's (penalised by how far its normal turns away from the meshlet's
  // mean normal) until it holds 64 triangles or 64 vertices.  Compact, connected patches: small bounding spheres
  // (fewer tiles per meshlet) and tight normal cones (more meshlets culled as back-facing).
  std::vector<char> assigned(F, 0), in_frontier(F, 0);
  std::vector<int> pending;  // faces that bordered a finished meshlet: preferred seeds (keeps neighbours together)
  size_t cursor = 0;         // Morton-order fallback for disconnected components
  int n_assigned = 0;
  std::vector<int> frontier;
  while (n_assigned < F) {
    int seed = -1;
    while (!pending.empty() && seed < 0) {
      const int f = pending.back();
      pending.pop_back();
      if (!assigned[f]) seed = f;
    }
    while (seed < 0) {
      const int f = order[cursor++];
      if (!assigned[f]) seed = f;
    }
    frontier.clear();
    V3 csum = {0, 0, 0}, nsum = {0, 0, 0};
    int next = seed;
    while (next >= 0) {
      const int f = next;
      const int i[3] = {faces[3 * f], faces[3 * f + 1], faces[3 * f + 2]};
      uint32_t packed = 0;
      for (int e = 0; e < 3; ++e) {
        if (slot_of[i[e]] < 0) {
          slot_of[i[e]] = (int)cur_verts.size();
          cur_verts.push_back(i[e]);
        }
        packed |= (uint32_t)slot_of[i[e]] << (8 * e);
      }
      cur_tris.push_back(make_uint2(packed, (unsigned)f));
      cur_faces.push_back(f);
      assigned[f] = 1;
      ++n_assigned;
      csum = {csum.x + fc[f].x, csum.y + fc[f].y, csum.z + fc[f].z};
      nsum = {nsum.x + fn[f].x, nsum.y + fn[f].y, nsum.z + fn[f].z};
      for (int a = adj_off[f]; a < adj_off[f + 1]; ++a) {
        const int g = adj[a];
        if (!assigned[g] && !in_frontier[g]) {
          in_frontier[g] = 1;
          frontier.push_back(g);
        }
      }
      next = -1;
      if ((int)cur_faces.size() == kMeshletTris) break;
      const double inv = 1.0 / cur_faces.size();
      const V3 ctr = {csum.x * inv, csum.y * inv, csum.z * inv};
      const double nl = norm(nsum);
      double best = 1e300;
      size_t best_k = 0;
      for (size_t k2 = 0; k2 < frontier.size(); ++k2) {
        const int g = frontier[k2];
        if (assigned[g]) continue;
        int fresh = 0;
        for (int e = 0; e < 3; ++e) {
          const int v = faces[3 * g + e];
          bool dup = false;
          for (int e2 = 0; e2 < e; ++e2) dup = dup || faces[3 * g + e2] == v;
          if (slot_of[v] < 0 && !dup) ++fresh;
        }
        if ((int)cur_verts.size() + fresh > kMeshletVerts) continue;
        const V3 dv = sub(fc[g], ctr);
        const double turn = nl > 1e-12 ? 1.0 - dot(fn[g], nsum) / nl : 0.0;  // 0 = parallel, 2 = opposite
        // faces about to be orphaned (no / one unassigned neighbour left) go first: fewer left-over islands
        int live = 0;
        for (int a = adj_off[g]; a < adj_off[g + 1]; ++a) live += !assigned[adj[a]];
        const double orphan = live == 0 ? 0.2 : (live == 1 ? 0.55 : 1.0);
        const double score = dot(dv, dv) * (1.0 + 2.0 * turn) * orphan + 1e-30 * fresh;
        if (score < best) {
          best = score;
          best_k = k2;
          next = g;
        }
      }
      if (next >= 0) {
        frontier[best_k] = frontier.back();
        frontier.pop_back();
        in_frontier[next] = 0;
      }
    }
    for (int g : frontier) {
      in_frontier[g] = 0;
      if (!assigned[g]) pending.push_back(g);
    }
    flush();
  }
  return 0;

}

}  // namespace fp
