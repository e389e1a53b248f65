/* octomap_oracle.c -- plain-C restatement of the colour OctoMap the reference writes (octomap 1.6-1.8, ColorOcTree as
 * ColorOctomapServer::insertCloudCallback drives it), rules 2-8 of DESIGN.md 4.14.  A literal pointer octree of 16 levels:
 *   - om_insert: one scan.  computeUpdate (free / occupied key sets, occupied winning), one updateNode per key (lazy: the leaf
 *     only, inner nodes are created empty), averageNodeColor per finite point in order, then updateInnerOccupancy.
 *   - om_write: AbstractOcTree::write into a buffer (header + pre-order 8-byte records).
 * Compile with -ffp-contract=off: octomap on x86-64 does not contract. */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define OM_DEPTH 16
#define OM_WHITE 0xffffffu

typedef struct Node {
  float lo;
  uint32_t rgb; /* r << 16 | g << 8 | b; OM_WHITE: unset */
  struct Node* child[8];
} Node;

typedef struct {
  double res, rf;
  float hit, miss, cmin, cmax;
  Node* root;
  long size; /* tree_size */
} Map;

typedef struct {
  uint16_t k[3];
} Key;

typedef struct {
  Key* v;
  long n, cap;
} Keys;

static void keys_push(Keys* s, const uint16_t k[3]) {
  if (s->n == s->cap) {
    s->cap = s->cap ? 2 * s->cap : 1024;
    s->v = (Key*)realloc(s->v, sizeof(Key) * s->cap);
  }
  memcpy(s->v[s->n++].k, k, 6);
}

static float logodds(double p) { return (float)log(p / (1 - p)); }

void* om_create(double res, double hit, double miss, double cmin, double cmax) {
  Map* m = (Map*)calloc(1, sizeof(Map));
  m->res = res;
  m->rf = 1.0 / res;
  m->hit = logodds(hit);
  m->miss = logodds(miss);
  m->cmin = logodds(cmin);
  m->cmax = logodds(cmax);
  return m;
}

static void free_rec(Node* n) {
  if (!n) return;
  for (int i = 0; i < 8; i++) free_rec(n->child[i]);
  free(n);
}

void om_clear(void* p) {
  Map* m = (Map*)p;
  free_rec(m->root);
  m->root = NULL;
  m->size = 0;
}

void om_destroy(void* p) {
  om_clear(p);
  free(p);
}

/* coordToKeyChecked */
static int key1(const Map* m, float c, uint16_t* k) {
  const double v = floor(m->rf * (double)c);
  if (!(v >= -32768.0 && v < 32768.0)) return 0;
  *k = (uint16_t)((int)v + 32768);
  return 1;
}
static int key3(const Map* m, const float p[3], uint16_t k[3]) {
  return key1(m, p[0], &k[0]) && key1(m, p[1], &k[1]) && key1(m, p[2], &k[2]);
}

/* computeRayKeys: appends the ray's cells; returns 0 when a key is out of range */
static int ray_keys(const Map* m, const float o[3], const float e[3], Keys* out) {
  uint16_t ko[3], ke[3];
  if (!key3(m, o, ko) || !key3(m, e, ke)) return 0;
  if (!memcmp(ko, ke, 6)) return 1;
  keys_push(out, ko);
  float d[3] = {e[0] - o[0], e[1] - o[1], e[2] - o[2]};
  const float len = (float)sqrt((double)(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]));
  for (int i = 0; i < 3; i++) d[i] /= len;
  int step[3];
  double tmax[3], tdelta[3];
  for (int i = 0; i < 3; i++) {
    step[i] = d[i] > 0.0 ? 1 : (d[i] < 0.0 ? -1 : 0);
    if (step[i] != 0) {
      double border = ((double)((int)ko[i] - 32768) + 0.5) * m->res;
      border += (float)(step[i] * m->res * 0.5);
      tmax[i] = (border - o[i]) / d[i];
      tdelta[i] = m->res / fabsf(d[i]);
    } else {
      tmax[i] = DBL_MAX;
      tdelta[i] = DBL_MAX;
    }
  }
  uint16_t cur[3] = {ko[0], ko[1], ko[2]};
  for (;;) {
    unsigned dim;
    if (tmax[0] < tmax[1]) dim = tmax[0] < tmax[2] ? 0 : 2;
    else dim = tmax[1] < tmax[2] ? 1 : 2;
    cur[dim] += step[dim];
    tmax[dim] += tdelta[dim];
    if (!memcmp(cur, ke, 6)) break;
    const double dist = fmin(fmin(tmax[0], tmax[1]), tmax[2]);
    if (dist > len) break;
    keys_push(out, cur);
  }
  return 1;
}

/* for the tests: the cells of one ray, -1 when a key is out of range */
long om_ray_keys(double res, const float* o, const float* e, uint16_t* out, long cap) {
  Map m;
  memset(&m, 0, sizeof(m));
  m.res = res;
  m.rf = 1.0 / res;
  Keys k = {0, 0, 0};
  const int ok = ray_keys(&m, o, e, &k);
  for (long i = 0; i < k.n && i < cap; i++) memcpy(out + 3 * i, k.v[i].k, 6);
  const long n = ok ? k.n : -1;
  free(k.v);
  return n;
}

static int child_idx(const uint16_t k[3], int bit) {
  return ((k[0] >> bit) & 1) | (((k[1] >> bit) & 1) << 1) | (((k[2] >> bit) & 1) << 2);
}

static Node* new_node(Map* m) {
  Node* n = (Node*)calloc(1, sizeof(Node));
  n->rgb = OM_WHITE;
  m->size++;
  return n;
}

/* updateNode(key, occupied, lazy_eval = true) */
static void update(Map* m, const uint16_t k[3], int occupied) {
  if (!m->root) m->root = new_node(m);
  Node* n = m->root;
  for (int d = OM_DEPTH - 1; d >= 0; d--) {
    const int c = child_idx(k, d);
    if (!n->child[c]) n->child[c] = new_node(m);
    n = n->child[c];
  }
  n->lo += occupied ? m->hit : m->miss;
  if (n->lo < m->cmin) n->lo = m->cmin;
  if (n->lo > m->cmax) n->lo = m->cmax;
}

static Node* search(const Map* m, const uint16_t k[3]) {
  Node* n = m->root;
  for (int d = OM_DEPTH - 1; n && d >= 0; d--) n = n->child[child_idx(k, d)];
  return n;
}

static int key_cmp(const void* a, const void* b) { return memcmp(a, b, 6); }

static long unique(Keys* s) {
  if (s->n == 0) return 0;
  qsort(s->v, s->n, sizeof(Key), key_cmp);
  long w = 1;
  for (long i = 1; i < s->n; i++)
    if (memcmp(s->v[i].k, s->v[w - 1].k, 6)) s->v[w++] = s->v[i];
  return s->n = w;
}

static void inner_rec(Node* n, int depth) {
  int has = 0;
  for (int i = 0; i < 8; i++) has |= n->child[i] != NULL;
  if (!has) return;
  if (depth < OM_DEPTH)
    for (int i = 0; i < 8; i++)
      if (n->child[i]) inner_rec(n->child[i], depth + 1);
  float mx = -FLT_MAX;
  int mr = 0, mg = 0, mb = 0, c = 0;
  for (int i = 0; i < 8; i++) {
    const Node* ch = n->child[i];
    if (!ch) continue;
    if (ch->lo > mx) mx = ch->lo;
    if (ch->rgb != OM_WHITE) {
      mr += ch->rgb >> 16;
      mg += (ch->rgb >> 8) & 0xff;
      mb += ch->rgb & 0xff;
      c++;
    }
  }
  n->lo = mx;
  n->rgb = c > 0 ? ((uint32_t)(mr / c) << 16) | ((uint32_t)(mg / c) << 8) | (uint32_t)(mb / c) : OM_WHITE;
}

/* One scan: xyz (n x 3 float, transformed), rgb (n colour words), origin, max_range (< 0: none).  Returns the number of
 * ray cells and occupied cells the scan produced, before the sets are formed. */
long om_insert(void* p, const float* xyz, const uint32_t* rgb, long n, const float* origin, double max_range) {
  Map* m = (Map*)p;
  Keys fr = {0, 0, 0}, oc = {0, 0, 0};
  for (long i = 0; i < n; i++) {
    const float* q = xyz + 3 * i;
    if (!isfinite(q[0]) || !isfinite(q[1]) || !isfinite(q[2])) continue;
    float d[3] = {q[0] - origin[0], q[1] - origin[1], q[2] - origin[2]};
    const double norm = sqrt((double)(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]));
    if (max_range < 0.0 || norm <= max_range) {
      ray_keys(m, origin, q, &fr);
      uint16_t k[3];
      if (key3(m, q, k)) keys_push(&oc, k);
    } else {
      if (norm > 0)
        for (int c = 0; c < 3; c++) d[c] /= (float)norm;
      float e[3];
      for (int c = 0; c < 3; c++) e[c] = origin[c] + d[c] * (float)max_range;
      ray_keys(m, origin, e, &fr);
    }
  }
  const long cells = fr.n + oc.n;
  unique(&fr);
  unique(&oc);
  for (long i = 0; i < fr.n; i++)
    if (!bsearch(fr.v[i].k, oc.v, oc.n, sizeof(Key), key_cmp)) update(m, fr.v[i].k, 0);
  for (long i = 0; i < oc.n; i++) update(m, oc.v[i].k, 1);
  free(fr.v);
  free(oc.v);
  for (long i = 0; i < n; i++) { /* averageNodeColor */
    const float* q = xyz + 3 * i;
    if (isnan(q[0]) || isnan(q[1]) || isnan(q[2])) continue;
    uint16_t k[3];
    if (!key3(m, q, k)) continue;
    Node* leaf = search(m, k);
    if (!leaf) continue;
    const uint32_t c = rgb[i] & 0xffffffu;
    if (leaf->rgb != OM_WHITE) {
      uint32_t o = 0;
      for (int s = 0; s < 24; s += 8) o |= ((((leaf->rgb >> s) & 0xff) + ((c >> s) & 0xff)) / 2) << s;
      leaf->rgb = o;
    } else {
      leaf->rgb = c;
    }
  }
  if (m->root) inner_rec(m->root, 0);
  return cells;
}

static void leaves_rec(const Node* n, int depth, long* leaves) {
  if (depth == OM_DEPTH) {
    (*leaves)++;
    return;
  }
  for (int i = 0; i < 8; i++)
    if (n->child[i]) leaves_rec(n->child[i], depth + 1, leaves);
}

void om_stats(void* p, long* nodes, long* leaves) {
  Map* m = (Map*)p;
  *nodes = m->size;
  *leaves = 0;
  if (m->root) leaves_rec(m->root, 0, leaves);
}

static uint8_t* write_rec(const Node* n, uint8_t* o) {
  uint8_t bits = 0;
  for (int i = 0; i < 8; i++)
    if (n->child[i]) bits |= (uint8_t)(1u << i);
  memcpy(o, &n->lo, 4);
  o[4] = (uint8_t)(n->rgb >> 16);
  o[5] = (uint8_t)(n->rgb >> 8);
  o[6] = (uint8_t)n->rgb;
  o[7] = bits;
  o += 8;
  for (int i = 0; i < 8; i++)
    if (n->child[i]) o = write_rec(n->child[i], o);
  return o;
}

/* The .ot bytes: returns their count; writes them when out holds cap >= that many. */
long om_write(void* p, uint8_t* out, long cap) {
  Map* m = (Map*)p;
  char head[256];
  const int h = snprintf(head, sizeof(head),
                         "# Octomap OcTree file\n# (feel free to add / change comments, but leave the first line as it is!)\n#\n"
                         "id ColorOcTree\nsize %ld\nres %g\ndata\n",
                         m->size, m->res);
  const long total = h + 8 * m->size;
  if (!out || cap < total) return total;
  memcpy(out, head, h);
  if (m->root) write_rec(m->root, out + h);
  return total;
}
