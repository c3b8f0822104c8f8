// ag_solver.cuh — K6 (constraint rows -> packed per-env row stream) and K7 (PGS over the stream).
//
// What it restates: Bullet's btMultiBodyConstraintSolver for one p.stepSimulation (envs/env.py:226):
// joint-limit rows (only while violated), joint-motor rows (agent.py:33), the spoon<->gripper fixed
// constraint (tool.py:46-47, 6 rows, maxForce 500) and frictional contacts (1 normal + 2 friction
// rows, implicit cone), solved by projected Gauss-Seidel in that order, 50 iterations, early exit on
// the least-squares residual.
//
// Design (round 2).  The Gauss-Seidel chain of one env is strictly sequential, so K7's speed is
// the latency and the instruction count of one row update; round 1 ran it on ONE lane per env
// (~450 cycles and ~115 warp instructions per row).  Now FOUR lanes cooperate on an env and a warp
// carries eight envs in lock-step:
//   * the env's velocity-delta vector lives in shared memory in 8-float blocks (one block per free
//     body, one or two per articulation); lane l of the env's lane group owns entries 8j + 2l and
//     8j + 2l + 1, so a row's J.v is two FMA chains per lane per block, one add and a 2-level
//     xor-shuffle reduction -- the same summation tree as one lane per entry --, and the update
//     v += M^-1 J^T dlambda is two FMAs per lane per block -- no cross-lane traffic through memory;
//   * K6 writes the rows as RECORDS in one env-major stream (HBM/L2): a 64 B header (indices, rhs,
//     1/diag, bounds) and up to four 128 B lane blocks, entry-major ([entry][J1 M1 J2 M2]), so a lane
//     fetches its share of a block with two LDS.128;
//   * a record carries TWO rows that act on the same pair of bodies: two consecutive box rows
//     (limit / motor / fixed-constraint / contact-normal) with their Gauss-Seidel coupling
//     w21 = J2 M^-1 J1^T precomputed by K6 (row 2 sees row 1's update through one scalar FMA, which
//     is algebraically the sequential sweep), or the two friction rows of a contact (solved jointly
//     against the cone).  Both rows share the loads and the shuffle reduction;
//   * the read-only stream flows through a 4 KB ring per env: the first tile by a TMA bulk copy
//     (cp.async.bulk + mbarrier complete_tx), then cp.async pieces right behind the consumer (see
//     pgs_warp); the next record's header and lane blocks are loaded while the current record is solved.
// Records never straddle a chunk (the packer pads).
#pragma once
#include "ag_device.cuh"

#define RS_HDR 16             // header floats (64 B)
#define RS_LB 32              // floats per lane block: 8 entries x [J1 M1 J2 M2] (128 B)
#define RS_UNIT 16            // record sizes / offsets are multiples of 16 floats
#define RS_MAXREC (RS_HDR + 4 * RS_LB)
// record modes
enum { RM_BOX = 0, RM_CONE = 1, RM_PAD = 2 };
// Header (ints are stored as raw bits; offsets are BYTE offsets from the start of the env's velocity block in K7's
// shared memory, where the impulses follow the velocities, so K7 forms an address with one add):
//   [0] nv | mode << 4 | (record bytes) << 8             nv = number of lane blocks (0..4)
//   [1] slot0 | slot1 << 16   [2] slot2 | slot3 << 16   each block's 8 entries in the velocity vector (4 * index)
//   [3] li1 | li2 << 16                                  the two rows' impulses (4 * (rs_nv + index))
//   [4] lin                                              RM_CONE: impulse of the contact's normal row
//   [5] w21   [6] mu   [7] -
//   [8..11] rhs1 dinv1 lo1 hi1   [12..15] rhs2 dinv2 lo2 hi2     (RM_CONE ignores lo/hi)
// Lane block k, quad i: [J1 M1 J2 M2] of velocity entry slot_k + i.  Unused slots point at the env's null block
// (8 zeros at the end of the velocity vector), an absent second row has li2 = the dummy impulse and all-zero data.

struct alignas(16) v4 { float x, y, z, w; };
AG_HD v4 ldv4(const float* p) { return *(const v4*)p; }
AG_HD void stv4(float* p, v4 a) { *(v4*)p = a; }
AG_HD float i2f_bits(int v) { float f; memcpy(&f, &v, 4); return f; }
AG_HD int f2i_bits(float f) { int v; memcpy(&v, &f, 4); return v; }

// velocity-delta vector of one env: [articulation a: its dofs padded to 8, at art_voff[a]]...[free body f: lin xyz, ang xyz, 2 pad][null block: 8 zeros]
AG_HD int rs_null(const SimDev& S) { return S.NDp + 8 * S.nf; }
AG_HD int rs_nv(const SimDev& S) { return (S.NDp + 8 * S.nf + 8 + 31) & ~31; }
// impulses: [3 ND dof rows][ngr fixed-constraint rows][3 per contact][dummy]
AG_HD int rs_dummy(const SimDev& S) { return 3 * S.ND + S.ngr + 3 * S.maxc; }
AG_HD int rs_nlam(const SimDev& S) { return (3 * S.ND + S.ngr + 3 * S.maxc + 1 + 31) & ~31; }
// shared memory of a K7 CTA (RS_CTA_ENVS envs): 4 KB alignment slack, per env the 4 KB stream ring, per env velocity
// deltas and impulses (stride rs_env_stride), one 8-byte mbarrier per env
#define RS_CTA_ENVS 8
AG_HD int rs_env_floats(const SimDev& S) { return rs_nv(S) + rs_nlam(S) + 64 + 1024; }      // (host emulation layout)
// +8 floats: consecutive envs' vectors start 32 B apart modulo 128 B, so the eight lane groups' 32-byte velocity accesses
// to the same entries fall into different banks
AG_HD int rs_env_stride(const SimDev& S) { return rs_nv(S) + rs_nlam(S) + 8; }
AG_HD int rs_cta_floats(const SimDev& S) { return 1024 + RS_CTA_ENVS * (1024 + rs_env_stride(S)) + 2 * RS_CTA_ENVS; }

// ------------------------------------------------------------------ K6: constraint rows
// side reference encoding: (idx << 2) | kind, kind: 0 static, 1 free body (idx = f), 2 articulated (idx = dyn link)
AG_HD int link_ref(const SimDev& S, int e, int link) {
  int b = AG_LDG(S.link_body + link);
  int kind = AG_LDG(S.body_kind + b);
  if (S.body_mode[(size_t)b * S.N + e] != 1) return 0;
  if (kind == BK_FREE) return (AG_LDG(S.body_idx + b) << 2) | 1;
  if (kind == BK_ART) { int d = AG_LDG(S.link_dl + link); return d < 0 ? 0 : ((d << 2) | 2); }
  return 0;
}

AG_HD s3 ld_Iinv(const SimDev& S, int f, int e) {
  size_t ib = (size_t)f * 6 * S.N + e; size_t N = S.N;
  s3 r; r.xx = S.fIinv[ib]; r.yy = S.fIinv[ib + N]; r.zz = S.fIinv[ib + 2 * N]; r.xy = S.fIinv[ib + 3 * N]; r.xz = S.fIinv[ib + 4 * N]; r.yz = S.fIinv[ib + 5 * N];
  return r;
}

// where a side's velocity entries live in the env's velocity-delta vector, and how many there are
AG_HD void side_dims(const SimDev& S, int ref, int& off, int& n) {
  int kind = ref & 3, idx = ref >> 2;
  if (kind == 1) { off = S.NDp + 8 * idx; n = 6; }
  else if (kind == 2) { int a = AG_LDG(S.dl_art + idx); off = AG_LDG(S.art_voff + a); n = AG_LDG(S.art_nd + a); }
  else { off = 0; n = 0; }
}
// side order of a record: a lone dynamic side is A, an articulation paired with a free body is A (J carries the sign)
AG_HD bool rs_swap_sides(int refA, int refB) {
  int ka = refA & 3, kb = refB & 3;
  return (ka == 0 && kb != 0) || (ka == 1 && kb == 2);
}

// The lane blocks of a record whose sides occupy (offA, nA) and (offB, nB): [A 0-7][A 8-15][B 0-7][B 8-15], absent ones
// dropped.  Two links of the SAME articulation (self-collision) share one set of blocks: side B accumulates into side A's.
struct RsShape { int nv, sl[4], slotB, offA, nA, offB, nB; bool merged; };
AG_HD RsShape rs_shape(const SimDev& S, int refA, int refB) {
  RsShape h;
  side_dims(S, refA, h.offA, h.nA); side_dims(S, refB, h.offB, h.nB);
  h.merged = h.nA > 0 && h.nB > 0 && h.offA == h.offB;
  const int null = rs_null(S);
  // blocks of A, then of B; every index into sl is a constant, so the shape stays in registers
  const int na = h.nA > 0 ? (h.nA > 8 ? 2 : 1) : 0, nb = (h.nB > 0 && !h.merged) ? (h.nB > 8 ? 2 : 1) : 0;
#pragma unroll
  for (int k = 0; k < 4; k++) h.sl[k] = k < na ? h.offA + 8 * k : (k < na + nb ? h.offB + 8 * (k - na) : null);
  h.nv = na + nb;
  h.slotB = h.merged ? 0 : na;
  return h;
}
AG_HD int rs_shape_key(const RsShape& h) { return h.nv == 0 ? -1 : (h.sl[0] | (h.merged ? 0x8000 : 0) | ((h.nB > 0 && !h.merged ? h.offB + 1 : 0) << 16)); }
AG_HD int rs_rec_floats(int nv) { return RS_HDR + RS_LB * nv; }
// header encodings
AG_HD int rs_enc_meta(int nv, int mode, int floats) { return nv | (mode << 4) | ((floats * 4) << 8); }
AG_HD int rs_enc_slot(int idx) { return idx * 4; }
AG_HD int rs_enc_lam(const SimDev& S, int li) { return (rs_nv(S) + li) * 4; }
AG_HD int rs_meta_floats(int meta) { return (meta >> 8) / 4; }

// address of (J, M) of entry i of the side whose first lane block is `slot0`, for row `row` (0 / 1) of record `rec`
AG_HD float* rs_entry(float* rec, int slot0, int i, int row) { return rec + RS_HDR + (slot0 + (i >> 3)) * RS_LB + (i & 7) * 4 + 2 * row; }

// One side of a row: unit force `lin` at world point p plus torque `ang`.  Writes (or, `acc`, adds) the side's J entries
// and M^-1 J^T into the record's lane blocks, accumulates J.v (pre-solve velocities) into rel.  Returns nothing: the
// row's diagonal J M^-1 J^T is taken from the finished blocks (rs_row_diag), which is also right for merged sides.
AG_HDN inline void emit_side(const SimDev& S, int e, int ref, f3 p, f3 lin, f3 ang, float* rec, int slot0, int row, bool acc, float& rel) {
  const int N = S.N;
  int kind = ref & 3, idx = ref >> 2;
  if (kind == 1) {
    int b = AG_LDG(S.free_body + idx);
    float invm = AG_LDG(S.free_invm + idx);
    f3 r = p - ld3(S.fcom, idx, N, e);
    f3 t = cross(r, lin) + ang;
    f3 it = mul(ld_Iinv(S, idx, e), t);
    f3 v = ld3(S.base_lin, b, N, e), w = ld3(S.base_ang, b, N, e);
    rel += dot(lin, v) + dot(t, w);
    float J[6] = {lin.x, lin.y, lin.z, t.x, t.y, t.z};
    float M[6] = {lin.x * invm, lin.y * invm, lin.z * invm, it.x, it.y, it.z};
    for (int i = 0; i < 6; i++) { float* d = rs_entry(rec, slot0, i, row); d[0] = J[i]; d[1] = M[i]; }
  } else if (kind == 2) {
    // J lives in registers: every index into it is a constant of the unrolled loops.  A dof's parent precedes it
    // (dyn_body's leaf-to-root pass relies on the same order), so one downward sweep meets the whole chain from idx.
    float J[AG_MAXND];
    int a = AG_LDG(S.dl_art + idx), d0 = AG_LDG(S.art_dl0 + a), nd = AG_LDG(S.art_nd + a);
    int j = idx;
#pragma unroll
    for (int i = AG_MAXND - 1; i >= 0; i--) {
      J[i] = 0.f;
      if (i < nd && d0 + i == j) {
        f3 axw = ld3(S.jax, j, N, e), o = ld3(S.jor, j, N, e);
        J[i] = (AG_LDG(S.dl_type + j) == 1) ? (dot(lin, cross(axw, p - o)) + dot(ang, axw)) : dot(lin, axw);
        j = AG_LDG(S.dl_parent + j);
      }
    }
    for (int i = 0; i < nd; i++) {
      float m = 0.f, Ji = 0.f;
#pragma unroll
      for (int k = 0; k < AG_MAXND; k++) {
        if (k < nd) m += S.Minv[((size_t)(d0 + i) * S.ND + (d0 + k)) * N + e] * J[k];
        if (k == i) Ji = J[k];
      }
      float* d = rs_entry(rec, slot0, i, row);
      if (acc) { d[0] += Ji; d[1] += m; } else { d[0] = Ji; d[1] = m; }
      rel += Ji * ld1(S.jqd, AG_LDG(S.dl_link + d0 + i), N, e);
    }
  }
}
// J M^-1 J^T of row `row`, and (row 1) the coupling J2 M^-1 J1^T, from the finished lane blocks
AG_HD float rs_row_diag(const float* rec, int nv, int row) {
  float d = 0.f;
  for (int i = 0; i < 8 * nv; i++) { const float* q = rec + RS_HDR + 4 * i + 2 * row; d += q[0] * q[1]; }
  return d;
}
AG_HD float rs_row_w21(const float* rec, int nv) {
  float d = 0.f;
  for (int i = 0; i < 8 * nv; i++) { const float* q = rec + RS_HDR + 4 * i; d += q[2] * q[1]; }
  return d;
}
AG_HD void rs_zero_blocks(float* rec, int nv) {
  v4 z; z.x = z.y = z.z = z.w = 0.f;
  for (int i = 0; i < 8 * nv; i++) stv4(rec + RS_HDR + 4 * i, z);
}
// structural part of a header + null second row; the rows' numbers are filled in by rs_set_row
AG_HD void rs_header(const SimDev& S, float* rec, const RsShape& h, int mode) {
  const int dummy = rs_dummy(S);
  rec[0] = i2f_bits(rs_enc_meta(h.nv, mode, rs_rec_floats(h.nv)));
  rec[1] = i2f_bits(rs_enc_slot(h.sl[0]) | (rs_enc_slot(h.sl[1]) << 16)); rec[2] = i2f_bits(rs_enc_slot(h.sl[2]) | (rs_enc_slot(h.sl[3]) << 16));
  rec[3] = i2f_bits(rs_enc_lam(S, dummy) | (rs_enc_lam(S, dummy) << 16)); rec[4] = i2f_bits(rs_enc_lam(S, dummy));
  for (int i = 5; i < RS_HDR; i++) rec[i] = 0.f;
}
AG_HD void rs_set_li(const SimDev& S, float* rec, int row, int li0) {
  const int li = rs_enc_lam(S, li0);
  int w = f2i_bits(rec[3]);
  w = row == 0 ? ((w & ~0xffff) | li) : ((w & 0xffff) | (li << 16));
  rec[3] = i2f_bits(w);
}
AG_HD void rs_set_row(const SimDev& S, float* rec, int row, int li, float rhs, float dinv, float lo, float hi) {
  rs_set_li(S, rec, row, li);
  float* d = rec + 8 + 4 * row;
  d[0] = rhs; d[1] = dinv; d[2] = lo; d[3] = hi;
}
// a row whose diagonal vanished (no motion possible along it): zero its J / M so it neither moves anything nor couples
AG_HD void rs_null_row(float* rec, int nv, int row) {
  for (int i = 0; i < 8 * nv; i++) { float* q = rec + RS_HDR + 4 * i + 2 * row; q[0] = 0.f; q[1] = 0.f; }
}

// stream allocator of K6a: reserve `nf` floats
struct RsCur { int pos; float* rs; int capf; bool over; };
AG_HD void rs_pad_header(const SimDev& S, float* rec, int mode, int floats) {
  const int null = rs_null(S), dummy = rs_dummy(S);
  rec[0] = i2f_bits(rs_enc_meta(0, mode, floats));
  rec[1] = i2f_bits(rs_enc_slot(null) | (rs_enc_slot(null) << 16)); rec[2] = rec[1];
  rec[3] = i2f_bits(rs_enc_lam(S, dummy) | (rs_enc_lam(S, dummy) << 16)); rec[4] = i2f_bits(rs_enc_lam(S, dummy));
  for (int i = 5; i < RS_HDR; i++) rec[i] = 0.f;
}
// word i of a null record's header (what rs_pad_header(S, rec, RM_BOX, 0) writes)
AG_HD float rs_null_word(const SimDev& S, int i) {
  const int null = rs_enc_slot(rs_null(S)), dummy = rs_enc_lam(S, rs_dummy(S));
  return i == 1 || i == 2 ? i2f_bits(null | (null << 16)) : (i == 3 ? i2f_bits(dummy | (dummy << 16)) : (i == 4 ? i2f_bits(dummy) : i2f_bits(0)));
}
AG_HD int rs_alloc(const SimDev&, RsCur& c, int nf) {
  if (c.pos + nf > c.capf) { c.over = true; return -1; }
  int o = c.pos; c.pos += nf;
  return o;
}
// row -> record map entries: (record offset / 16) << 2 | has-partner << 1 | position in the record
AG_HD int rs_enc(int off, int pos, int partner) { return ((off / RS_UNIT) << 2) | (partner << 1) | pos; }

// Is dof row r = kind * ND + d (kind 0 lower limit, 1 upper limit, 2 motor) live this substep?  If so: its constants.
struct DofRow { float rhs, dinv, lo, hi, sgn; };
AG_HD bool dof_row(const SimDev& S, int e, int kind, int d, DofRow& R) {
  const int N = S.N;
  const float dt = S.dt;
  int k = AG_LDG(S.dl_link + d);
  float Mdd = S.Minv[((size_t)d * S.ND + d) * N + e];
  if (!(Mdd > 0.f)) return false;
  R.dinv = 1.0f / Mdd; R.lo = 0.f; R.hi = 1e30f; R.sgn = 1.f;
  float q = ld1(S.jq, k, N, e), qd = ld1(S.jqd, k, N, e);
  if (kind < 2) {             // limits: a row only while violated
    if (!AG_LDG(S.link_haslimit + k)) return false;
    if (kind == 0) { float pen = q - AG_LDG(S.link_lower + k); if (pen > 0.f) return false; R.rhs = (-pen * S.erp / dt - qd) * R.dinv; }
    else { float pen = AG_LDG(S.link_upper + k) - q; if (pen > 0.f) return false; R.rhs = (-pen * S.erp / dt + qd) * R.dinv; R.sgn = -1.f; }
  } else {
    int mode = S.motor_mode[k];
    float maxi = S.motor_maxf[k] * dt;
    if (S.motor_fscale) maxi *= ld1(S.motor_fscale, k, N, e);
    if (mode == 0 || !(maxi > 0.f)) return false;
    float vt = (mode == 1) ? (S.motor_kp[k] * (ld1(S.motor_target, k, N, e) - q) / dt + qd - S.motor_kd[k] * qd)
                           : ld1(S.motor_target, k, N, e);
    R.rhs = (vt - qd) * R.dinv; R.lo = -maxi; R.hi = maxi;
  }
  return true;
}
// sides of fixed constraint c in record order (articulation / lone dynamic side first)
AG_HD bool con_sides(const SimDev& S, int e, int c, int& refA, int& refB, bool& swapped) {
  const int N = S.N;
  int ka = AG_LDG(S.con_link + 2 * c), kb = AG_LDG(S.con_link + 2 * c + 1);
  int ba = AG_LDG(S.link_body + ka), bb = AG_LDG(S.link_body + kb);
  if (S.body_mode[(size_t)ba * N + e] == 0 || S.body_mode[(size_t)bb * N + e] == 0) return false;
  refA = link_ref(S, e, ka); refB = link_ref(S, e, kb);
  swapped = rs_swap_sides(refA, refB);
  if (swapped) { int t = refA; refA = refB; refB = t; }
  return ((refA | refB) & 3) != 0;
}

// Sides of contact `key` in record order; called by K4 for every sorted contact (one thread each) so that K6a's
// sequential pass only reads two ints per contact.
AG_HD void contact_refs(const SimDev& S, int e, unsigned key, int& refA, int& refB) {
  unsigned pairk = key >> 2;
  int ca = (int)(pairk / (unsigned)S.nc), cb = (int)(pairk % (unsigned)S.nc);
  refA = link_ref(S, e, AG_LDG(S.col_link + ca)); refB = link_ref(S, e, AG_LDG(S.col_link + cb));
  if (rs_swap_sides(refA, refB)) { int t = refA; refA = refB; refB = t | (1 << 30); }   // bit 30 of refB: sides were swapped
}

// K6a: one lane per env: the layout of this substep's row stream in solver order -- joint-limit rows (per dof: lower,
// upper), motor rows, fixed-constraint rows, contact normal rows (contact order), friction pairs (contact order) -- and
// which consecutive rows share a record.  Cheap and sequential; the records themselves are written by K6b.
// row_off [3 ND + ngr][N], s_ref[..][2]: rs_enc of each dof / fixed-constraint / contact-normal row (-1: not live);
// row_pair [3 ND + ngr][N]: the row that shares the record of a first row; s_ref[..][3]: friction record offset / 16.
AG_HDN inline void rows_body(int e, const SimDev& S, const KP&) {
  const int N = S.N;
  RsCur c; c.pos = 0; c.rs = S.rs_data + (size_t)e * S.rs_cap; c.capf = S.rs_cap; c.over = false;
  int open_key = -1, open_row = -1, open_off = -1;       // a record that still has room for a second row
  // ---- dof rows
  for (int pass = 0; pass < 2; pass++) {
    for (int d = 0; d < S.ND; d++) {
      for (int kind = (pass == 0 ? 0 : 2); kind < (pass == 0 ? 2 : 3); kind++) {
        const int r = kind * S.ND + d;
        DofRow R;
        int info = -1;
        if (dof_row(S, e, kind, d, R)) {
          int a = AG_LDG(S.dl_art + d);
          int key = 0x10000 | a;
          if (open_key == key) {
            info = rs_enc(open_off, 1, 1);
            S.row_off[(size_t)open_row * N + e] |= 2; S.row_pair[(size_t)open_row * N + e] = r;
            open_key = -1;
          } else {
            int nd = AG_LDG(S.art_nd + a);
            int o = rs_alloc(S, c, rs_rec_floats(nd > 8 ? 2 : 1));
            if (o >= 0) { info = rs_enc(o, 0, 0); open_key = key; open_row = r; open_off = o; }
          }
        }
        S.row_off[(size_t)r * N + e] = info;
        S.row_pair[(size_t)r * N + e] = -1;
      }
    }
  }
  open_key = -1;
  // ---- fixed constraints: rows (0,1) (2,3) (4,5) share records
  for (int cc = 0; cc < S.ncon; cc++) {
    int refA, refB; bool sw;
    bool on = con_sides(S, e, cc, refA, refB, sw);
    RsShape h; h.nv = 0;
    if (on) h = rs_shape(S, refA, refB);
    for (int i = 0; i < 6; i += 2) {
      int r = 3 * S.ND + 6 * cc + i;
      int i0 = -1, i1 = -1;
      if (on && h.nv > 0) {
        int o = rs_alloc(S, c, rs_rec_floats(h.nv));
        if (o >= 0) { i0 = rs_enc(o, 0, 1); i1 = rs_enc(o, 1, 1); }
      }
      S.row_off[(size_t)r * N + e] = i0; S.row_off[(size_t)(r + 1) * N + e] = i1;
      S.row_pair[(size_t)r * N + e] = i0 >= 0 ? r + 1 : -1; S.row_pair[(size_t)(r + 1) * N + e] = -1;
    }
  }
  // ---- contacts: normal rows (two consecutive contacts between the same bodies share a record), then friction pairs
  int cnt = S.c_count[e]; if (cnt > S.maxc) cnt = S.maxc;
  int open_slot = -1;
  for (int s = 0; s < cnt; s++) {
    size_t rb = (size_t)s * 4 * N + e;
    int refA = S.s_ref[rb], refB = S.s_ref[rb + N] & ~(1 << 30);     // written by K4 (contact_refs), bit 30 = sides swapped
    RsShape h = rs_shape(S, refA, refB);
    int key = rs_shape_key(h);
    int info = -1;
    if (key >= 0) {
      if (open_key == key && open_slot == s - 1) {
        info = rs_enc(open_off, 1, 1);
        S.s_ref[(size_t)(s - 1) * 4 * N + e + 2 * (size_t)N] |= 2;
        open_key = -1;
      } else {
        int o = rs_alloc(S, c, rs_rec_floats(h.nv));
        if (o >= 0) { info = rs_enc(o, 0, 0); open_key = key; open_slot = s; open_off = o; }
      }
    } else open_key = -1;
    S.s_ref[rb + 2 * (size_t)N] = info;
  }
  for (int s = 0; s < cnt; s++) {
    size_t rb = (size_t)s * 4 * N + e;
    int refA = S.s_ref[rb], refB = S.s_ref[rb + N] & ~(1 << 30);
    RsShape h = rs_shape(S, refA, refB);
    int o = -1;
    if (h.nv > 0 && S.s_ref[rb + 2 * (size_t)N] >= 0) o = rs_alloc(S, c, rs_rec_floats(h.nv));
    S.s_ref[rb + 3 * (size_t)N] = o < 0 ? -1 : o / RS_UNIT;
  }
  if (c.pos % 32 != 0) {                            // K7 refills its ring in 32-float pieces: pad with a null record
    if (c.pos + RS_UNIT <= c.capf) { rs_pad_header(S, c.rs + c.pos, RM_PAD, RS_UNIT); c.pos += RS_UNIT; } else c.over = true;
  }
  S.rs_nfloats[e] = c.over ? (c.pos / 32) * 32 : c.pos;
  if (c.over) S.overflow[e] = 1;
}

// finish a box row after its sides were emitted: diagonal, rhs, bounds; a vanishing diagonal nulls the row
AG_HD void rs_finish_box(const SimDev& S, float* rec, int nv, int row, int li, float num, float lo, float hi) {
  float diag = rs_row_diag(rec, nv, row);
  if (diag > 1e-20f) { float dinv = 1.0f / diag; rs_set_row(S, rec, row, li, num * dinv, dinv, lo, hi); }
  else rs_null_row(rec, nv, row);
}

// K6b, rows part: thread = (dof / fixed-constraint row r, env): the thread of a record's FIRST row builds the whole record
// in `rec` (see crows_record)
AG_HDN inline int drow_body(int r, int e, const SimDev& S, float* rec, float*& dst) {
  const int N = S.N;
  const float dt = S.dt;
  int info = S.row_off[(size_t)r * N + e];
  if (info < 0 || (info & 1)) return 0;
  dst = S.rs_data + (size_t)e * S.rs_cap + (size_t)(info >> 2) * RS_UNIT;
  const int r2 = (info & 2) ? S.row_pair[(size_t)r * N + e] : -1;
  if (r < 3 * S.ND) {
    int d = r % S.ND;
    int a = AG_LDG(S.dl_art + d), d0 = AG_LDG(S.art_dl0 + a), nd = AG_LDG(S.art_nd + a), vo = AG_LDG(S.art_voff + a);
    RsShape h; h.nv = nd > 8 ? 2 : 1; h.sl[0] = vo; h.sl[1] = nd > 8 ? vo + 8 : rs_null(S); h.sl[2] = h.sl[3] = rs_null(S);
    rs_header(S, rec, h, RM_BOX);
    rs_zero_blocks(rec, h.nv);
    int dd[2] = {d, 0}; float sg[2] = {1.f, 1.f};
#pragma unroll
    for (int row = 0; row < 2; row++) {
      if (row == 1 && r2 < 0) break;
      int rr = row == 0 ? r : r2;
      int kind = rr / S.ND; dd[row] = rr % S.ND;
      DofRow R;
      if (!dof_row(S, e, kind, dd[row], R)) continue;         // cannot happen: K6a saw the same state
      sg[row] = R.sgn;
      for (int i = 0; i < nd; i++) {
        float* q = rs_entry(rec, 0, i, row);
        q[0] = (i == dd[row] - d0) ? R.sgn : 0.f;
        q[1] = R.sgn * S.Minv[((size_t)(d0 + i) * S.ND + dd[row]) * N + e];
      }
      rs_set_row(S, rec, row, rr, R.rhs, R.dinv, R.lo, R.hi);
    }
    if (r2 >= 0) rec[5] = sg[0] * sg[1] * S.Minv[((size_t)dd[1] * S.ND + dd[0]) * N + e];
    return rs_rec_floats(h.nv);
  }
  // fixed constraint c, rows i and i + 1: 3 translation + 3 rotation rows
  int c = (r - 3 * S.ND) / 6, i0 = (r - 3 * S.ND) % 6;
  int refA, refB; bool sw;
  if (!con_sides(S, e, c, refA, refB, sw)) return 0;
  RsShape h = rs_shape(S, refA, refB);
  rs_header(S, rec, h, RM_BOX);
  rs_zero_blocks(rec, h.nv);
  int ka = AG_LDG(S.con_link + 2 * c), kb = AG_LDG(S.con_link + 2 * c + 1);
  q4 qa = ld4(S.lquat, ka, N, e), qb = ld4(S.lquat, kb, N, e);
  f3 pa = ld3(S.lpos, ka, N, e) + qrot(qa, tv3(S.con_pivot, 2 * c));
  f3 pb = ld3(S.lpos, kb, N, e) + qrot(qb, tv3(S.con_pivot, 2 * c + 1));
  f3 perr = pa - pb;
  q4 fa = qmul(qa, tv4(S.con_quat, 2 * c)), fb = qmul(qb, tv4(S.con_quat, 2 * c + 1));
  q4 qe = qmul(fa, qconj(fb));
  if (qe.w < 0.f) qe = q4(-qe.x, -qe.y, -qe.z, -qe.w);
  f3 aerr(2.f * qe.x, 2.f * qe.y, 2.f * qe.z);
  float sg = 1.f;
  if (sw) { f3 tp = pa; pa = pb; pb = tp; sg = -1.f; }     // the errors were measured before the swap: J is unchanged by it
  float maxi = AG_LDG(S.con_maxforce + c) * dt;
  for (int row = 0; row < (r2 >= 0 ? 2 : 1); row++) {
    int i = i0 + row;
    float err = i < 3 ? comp(perr, i) : comp(aerr, i - 3);
    f3 axv(i % 3 == 0 ? 1.f : 0.f, i % 3 == 1 ? 1.f : 0.f, i % 3 == 2 ? 1.f : 0.f);
    f3 lin = i < 3 ? axv : f3(), ang = i < 3 ? f3() : axv;
    float rel = 0.f;
    emit_side(S, e, refA, pa, lin * sg, ang * sg, rec, 0, row, false, rel);
    emit_side(S, e, refB, pb, lin * (-sg), ang * (-sg), rec, h.slotB, row, h.merged, rel);
    rs_finish_box(S, rec, h.nv, row, r + row, -err * S.erp / dt - rel, -maxi, maxi);
  }
  if (r2 >= 0) rec[5] = rs_row_w21(rec, h.nv);
  return rs_rec_floats(h.nv);
}

// ---- K6b fast path: records whose sides are free bodies (or static): both rows are built in registers.
struct FreeSide { float J[6], M[6], rel; };
AG_HD FreeSide free_side_zero() { FreeSide r; for (int i = 0; i < 6; i++) { r.J[i] = 0.f; r.M[i] = 0.f; } r.rel = 0.f; return r; }
// unit force `lin` at world point p on free body `idx` (side reference kind 1); anything else: zeros
AG_HD FreeSide free_side(const SimDev& S, int e, int ref, f3 p, f3 lin) {
  FreeSide r = free_side_zero();
  if ((ref & 3) != 1) return r;
  const int N = S.N, idx = ref >> 2;
  int b = AG_LDG(S.free_body + idx);
  float invm = AG_LDG(S.free_invm + idx);
  f3 t = cross(p - ld3(S.fcom, idx, N, e), lin);
  f3 it = mul(ld_Iinv(S, idx, e), t);
  f3 v = ld3(S.base_lin, b, N, e), w = ld3(S.base_ang, b, N, e);
  r.rel = dot(lin, v) + dot(t, w);
  r.J[0] = lin.x; r.J[1] = lin.y; r.J[2] = lin.z; r.J[3] = t.x; r.J[4] = t.y; r.J[5] = t.z;
  r.M[0] = lin.x * invm; r.M[1] = lin.y * invm; r.M[2] = lin.z * invm; r.M[3] = it.x; r.M[4] = it.y; r.M[5] = it.z;
  return r;
}
AG_HD float fs_dot(const FreeSide& a, const FreeSide& b) {        // a.J . b.M
  float d = 0.f;
  for (int i = 0; i < 6; i++) d += a.J[i] * b.M[i];
  return d;
}
AG_HD void rs_put_free_block(float* blk, const FreeSide& r1, const FreeSide& r2) {
  for (int i = 0; i < 6; i++) { v4 q; q.x = r1.J[i]; q.y = r1.M[i]; q.z = r2.J[i]; q.w = r2.M[i]; stv4(blk + 4 * i, q); }
  v4 z; z.x = z.y = z.z = z.w = 0.f;
  stv4(blk + 24, z); stv4(blk + 28, z);
}
// header of a record in registers
struct RsHead { float w[RS_HDR]; };
AG_HD RsHead rs_head(const SimDev& S, const RsShape& h, int mode) {
  RsHead H;
  const int dummy = rs_enc_lam(S, rs_dummy(S));
  H.w[0] = i2f_bits(rs_enc_meta(h.nv, mode, rs_rec_floats(h.nv)));
  H.w[1] = i2f_bits(rs_enc_slot(h.sl[0]) | (rs_enc_slot(h.sl[1]) << 16)); H.w[2] = i2f_bits(rs_enc_slot(h.sl[2]) | (rs_enc_slot(h.sl[3]) << 16));
  H.w[3] = i2f_bits(dummy | (dummy << 16)); H.w[4] = i2f_bits(dummy);
  for (int i = 5; i < RS_HDR; i++) H.w[i] = 0.f;
  return H;
}
AG_HD void rs_head_row(const SimDev& S, RsHead& H, int row, int li0, float rhs, float dinv, float lo, float hi) {
  const int li = rs_enc_lam(S, li0);
  int w = f2i_bits(H.w[3]);
  w = row == 0 ? ((w & ~0xffff) | li) : ((w & 0xffff) | (li << 16));
  H.w[3] = i2f_bits(w);
  H.w[8 + 4 * row] = rhs; H.w[9 + 4 * row] = dinv; H.w[10 + 4 * row] = lo; H.w[11 + 4 * row] = hi;
}
AG_HD void rs_head_store(float* rec, const RsHead& H) {
  for (int i = 0; i < 4; i++) { v4 q; q.x = H.w[4 * i]; q.y = H.w[4 * i + 1]; q.z = H.w[4 * i + 2]; q.w = H.w[4 * i + 3]; stv4(rec + 4 * i, q); }
}

// K6b: thread = (row, env): rows [0, maxc) are the sorted contacts, rows [maxc, maxc + 3 ND + ngr) the dof and
// fixed-constraint rows.  The thread of contact s writes the normal record that STARTS at s (one or two rows), part 0,
// and the friction record of s, part 1.  A part is built whole in `rec` (RS_MAXREC floats, 16-byte aligned, private to
// the thread); the return value is its length in floats (0: nothing to write) and `dst` its place in the stream.  The
// caller copies it there (k_crows: a warp stores its lanes' records as consecutive 16-byte pieces).
AG_HDN inline int crows_record(int tid, const SimDev& S, int part, float* rec, float*& dst) {
  const int N = S.N;
  int e = tid % N, slot = tid / N;
  if (slot >= S.maxc) return part == 0 ? drow_body(slot - S.maxc, e, S, rec, dst) : 0;
  int cnt = S.c_count[e]; if (cnt > S.maxc) cnt = S.maxc;
  if (slot >= cnt) return 0;
  if (part == 0) for (int d = 0; d < 3; d++) cf_st(S.s_data, slot, CF_LAM_N + d, N, e, 0.f);
  size_t rb = (size_t)slot * 4 * N + e;
  const int refA = S.s_ref[rb], refB0 = S.s_ref[rb + N], info = S.s_ref[rb + 2 * (size_t)N], of = S.s_ref[rb + 3 * (size_t)N];
  if (info < 0) return 0;
  const int refB = refB0 & ~(1 << 30);
  const RsShape h = rs_shape(S, refA, refB);
  float* rs = S.rs_data + (size_t)e * S.rs_cap;
  const float dt = S.dt;
  const int lam0 = 3 * S.ND + S.ngr;
  const bool fast = (refA & 3) == 1 && (refB & 3) != 2;      // sides: a free body and (nothing | a free body)
  if (part == 0) {
    if (info & 1) return 0;
    dst = rs + (size_t)(info >> 2) * RS_UNIT;
    const int nrow = (info & 2) ? 2 : 1;
    if (fast) {
      RsHead H = rs_head(S, h, RM_BOX);
      FreeSide a[2], b[2];
      a[1] = free_side_zero(); b[1] = free_side_zero();
#pragma unroll
      for (int row = 0; row < 2; row++) {
        if (row >= nrow) break;
        const int s = slot + row;
        f3 pa(cf_ld(S.s_data, s, CF_PAX, N, e), cf_ld(S.s_data, s, CF_PAY, N, e), cf_ld(S.s_data, s, CF_PAZ, N, e));
        f3 pb(cf_ld(S.s_data, s, CF_PBX, N, e), cf_ld(S.s_data, s, CF_PBY, N, e), cf_ld(S.s_data, s, CF_PBZ, N, e));
        f3 n(cf_ld(S.s_data, s, CF_NX, N, e), cf_ld(S.s_data, s, CF_NY, N, e), cf_ld(S.s_data, s, CF_NZ, N, e));
        float dist = cf_ld(S.s_data, s, CF_DIST, N, e);
        const int rA = S.s_ref[(size_t)s * 4 * N + e], rB0 = S.s_ref[(size_t)s * 4 * N + e + N];
        float sg = 1.f;
        if (rB0 & (1 << 30)) { f3 tp = pa; pa = pb; pb = tp; sg = -1.f; }
        a[row] = free_side(S, e, rA, pa, n * sg); b[row] = free_side(S, e, rB0 & ~(1 << 30), pb, n * (-sg));
        float diag = fs_dot(a[row], a[row]) + fs_dot(b[row], b[row]);
        float rel = a[row].rel + b[row].rel;
        float pen = dist + S.slop;
        float poserr, velerr = -rel;
        if (pen > 0.f) { poserr = 0.f; velerr -= pen / dt; } else poserr = -pen * S.contact_erp / dt;
        if (diag > 1e-20f) { float dinv = 1.0f / diag; rs_head_row(S, H, row, lam0 + 3 * s, (poserr + velerr) * dinv, dinv, 0.f, 1e30f); }
        else { a[row] = free_side_zero(); b[row] = free_side_zero(); }
      }
      if (nrow == 2) H.w[5] = fs_dot(a[1], a[0]) + fs_dot(b[1], b[0]);
      rs_head_store(rec, H);
      rs_put_free_block(rec + RS_HDR, a[0], a[1]);
      if (h.nv > 1) rs_put_free_block(rec + RS_HDR + RS_LB, b[0], b[1]);
    } else {
      rs_header(S, rec, h, RM_BOX);
      rs_zero_blocks(rec, h.nv);
      for (int row = 0; row < nrow; row++) {
        const int s = slot + row;
        f3 pa(cf_ld(S.s_data, s, CF_PAX, N, e), cf_ld(S.s_data, s, CF_PAY, N, e), cf_ld(S.s_data, s, CF_PAZ, N, e));
        f3 pb(cf_ld(S.s_data, s, CF_PBX, N, e), cf_ld(S.s_data, s, CF_PBY, N, e), cf_ld(S.s_data, s, CF_PBZ, N, e));
        f3 n(cf_ld(S.s_data, s, CF_NX, N, e), cf_ld(S.s_data, s, CF_NY, N, e), cf_ld(S.s_data, s, CF_NZ, N, e));
        float dist = cf_ld(S.s_data, s, CF_DIST, N, e);
        // the row's own sides (the partner contact touches the same bodies, but maybe other links of an articulation);
        // K4 may have swapped them (rs_swap_sides): the J entries carry the sign
        const int rA = S.s_ref[(size_t)s * 4 * N + e], rB0 = S.s_ref[(size_t)s * 4 * N + e + N];
        float sg = 1.f;
        if (rB0 & (1 << 30)) { f3 tp = pa; pa = pb; pb = tp; sg = -1.f; }
        float rel = 0.f;
        emit_side(S, e, rA, pa, n * sg, f3(), rec, 0, row, false, rel);
        emit_side(S, e, rB0 & ~(1 << 30), pb, n * (-sg), f3(), rec, h.slotB, row, h.merged, rel);
        float pen = dist + S.slop;
        float poserr, velerr = -rel;
        if (pen > 0.f) { poserr = 0.f; velerr -= pen / dt; } else poserr = -pen * S.contact_erp / dt;
        rs_finish_box(S, rec, h.nv, row, lam0 + 3 * s, poserr + velerr, 0.f, 1e30f);
      }
      if (nrow == 2) rec[5] = rs_row_w21(rec, h.nv);
    }
    return rs_rec_floats(h.nv);
  }
  if (of >= 0) {
    dst = rs + (size_t)of * RS_UNIT;
    f3 pa(cf_ld(S.s_data, slot, CF_PAX, N, e), cf_ld(S.s_data, slot, CF_PAY, N, e), cf_ld(S.s_data, slot, CF_PAZ, N, e));
    f3 pb(cf_ld(S.s_data, slot, CF_PBX, N, e), cf_ld(S.s_data, slot, CF_PBY, N, e), cf_ld(S.s_data, slot, CF_PBZ, N, e));
    f3 n(cf_ld(S.s_data, slot, CF_NX, N, e), cf_ld(S.s_data, slot, CF_NY, N, e), cf_ld(S.s_data, slot, CF_NZ, N, e));
    float sg = 1.f;
    if (refB0 & (1 << 30)) { f3 tp = pa; pa = pb; pb = tp; sg = -1.f; }
    unsigned pairk = S.s_key[(size_t)slot * N + e] >> 2;
    int ka = AG_LDG(S.col_link + (int)(pairk / (unsigned)S.nc)), kb = AG_LDG(S.col_link + (int)(pairk % (unsigned)S.nc));
    float mu = ld1(S.friction, ka, N, e) * ld1(S.friction, kb, N, e);
    f3 t1, t2; plane_space(n, t1, t2);
    if (fast) {
      RsHead H = rs_head(S, h, RM_CONE);
      FreeSide a[2], b[2];
#pragma unroll
      for (int row = 0; row < 2; row++) {
        f3 t = row == 0 ? t1 : t2;
        a[row] = free_side(S, e, refA, pa, t * sg); b[row] = free_side(S, e, refB, pb, t * (-sg));
        float diag = fs_dot(a[row], a[row]) + fs_dot(b[row], b[row]);
        float rel = a[row].rel + b[row].rel;
        if (diag > 1e-20f) { float dinv = 1.0f / diag; rs_head_row(S, H, row, lam0 + 3 * slot + 1 + row, -rel * dinv, dinv, 0.f, 0.f); }
        else { a[row] = free_side_zero(); b[row] = free_side_zero(); rs_head_row(S, H, row, lam0 + 3 * slot + 1 + row, 0.f, 0.f, 0.f, 0.f); }
      }
      H.w[4] = i2f_bits(rs_enc_lam(S, lam0 + 3 * slot)); H.w[6] = mu;
      rs_head_store(rec, H);
      rs_put_free_block(rec + RS_HDR, a[0], a[1]);
      if (h.nv > 1) rs_put_free_block(rec + RS_HDR + RS_LB, b[0], b[1]);
    } else {
      rs_header(S, rec, h, RM_CONE);
      rs_zero_blocks(rec, h.nv);
      for (int row = 0; row < 2; row++) {
        f3 t = row == 0 ? t1 : t2;
        float rel = 0.f;
        emit_side(S, e, refA, pa, t * sg, f3(), rec, 0, row, false, rel);
        emit_side(S, e, refB, pb, t * (-sg), f3(), rec, h.slotB, row, h.merged, rel);
        float diag = rs_row_diag(rec, h.nv, row);
        if (diag > 1e-20f) { float dinv = 1.0f / diag; rs_set_row(S, rec, row, lam0 + 3 * slot + 1 + row, -rel * dinv, dinv, 0.f, 0.f); }
        else { rs_null_row(rec, h.nv, row); rs_set_li(S, rec, row, lam0 + 3 * slot + 1 + row); }
      }
      rec[4] = i2f_bits(rs_enc_lam(S, lam0 + 3 * slot)); rec[6] = mu;
    }
    return rs_rec_floats(h.nv);
  }
  return 0;
}

// ------------------------------------------------------------------ K6c: heaviest-first env order for K7
// The PGS chain of an env is sequential and its length varies 10x between envs (iterations used x
// rows); the eight envs of a K7 warp run in lock-step, so envs of similar weight share a warp and the
// heaviest warps are issued first.  Work is predicted from this substep's stream length and the
// previous substep's iteration count.  One CTA: 64-bucket counting sort in shared memory.
AG_HD int pgs_work_bucket(const SimDev& S, int e) {
  int it = S.iters_used[e]; if (it < 1) it = 1;
  int w = it * (S.rs_nfloats[e] / 64);
  int b = 63 - w / 160;                               // heaviest work -> bucket 0
  return b < 0 ? 0 : b;
}

// ------------------------------------------------------------------ K7: PGS over the row stream
// The two rows of a record, given J1.v and J2.v (p1, p2) and the current impulses: new impulses and their changes.
struct RsSol { float s1, s2, d1, d2; };
// Branch-free on the device: the eight envs of a warp are at records of different modes, and a divergent branch in
// front of the warp-wide shuffles costs more than the few selects.  Everything that does not depend on p1 / p2 (the
// reduced J.v) is computed ahead of them: the dependent chain is fma, max, min, sub, fma, fma, max, min, sub.
// `dead`: the env has finished; the record is consumed without effect (bounds collapse onto the current impulses).
AG_HD RsSol rs_solve2(int mode, bool cone_cfg, bool dead, float p1, float p2, float lam1, float lam2, float lamn, const v4& ha, const v4& hb, float w21, float mu) {
  const bool cone_rec = mode == RM_CONE;
  const float lim = mu * lamn;
  const float big = 3.0e38f;
  const float bnd = cone_cfg ? big : lim;
  float lo1 = cone_rec ? -bnd : ha.z, hi1 = cone_rec ? bnd : ha.w, lo2 = cone_rec ? -bnd : hb.z, hi2 = cone_rec ? bnd : hb.w;
  lo1 = dead ? lam1 : lo1; hi1 = dead ? lam1 : hi1; lo2 = dead ? lam2 : lo2; hi2 = dead ? lam2 : hi2;
  const float a1 = lam1 + ha.x, a2 = lam2 + hb.x, lim2 = lim * lim;
  const bool can_scale = cone_rec && cone_cfg && !dead;
  RsSol r;
  float c1 = fminf(fmaxf(a1 - p1 * ha.y, lo1), hi1);
  float d1 = c1 - lam1;                                          // (a cone record has w21 = 0)
  float c2 = fminf(fmaxf(a2 - (p2 + w21 * d1) * hb.y, lo2), hi2);
  const float m2 = c1 * c1 + c2 * c2;
  const bool scale = can_scale && m2 > lim2;
#if defined(__CUDA_ARCH__)
  float rq; asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(rq) : "f"(m2));     // (scale => m2 > lim^2 >= 0; a denormal m2 cannot exceed a normal lim^2, and lim = 0 with a denormal m2 gives 0 * big = 0)
  const float kk = scale ? lim * rq : 1.0f;
#else
  const float kk = scale ? lim / sqrtf(m2) : 1.0f;
#endif
  c1 = scale ? c1 * kk : c1; c2 = scale ? c2 * kk : c2;
  r.d1 = c1 - lam1;
  r.d2 = c2 - lam2;
  r.s1 = c1; r.s2 = c2;
  return r;
}

#if defined(__CUDACC__)
typedef unsigned rs_addr;
__device__ __forceinline__ rs_addr rs_smem_addr(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void rs_bar_init(rs_addr bar) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(bar) : "memory");
}
__device__ __forceinline__ void rs_expect(rs_addr bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory");
}
// one TMA bulk copy global -> shared, completion counted in bytes on `bar`
__device__ __forceinline__ void rs_fetch(rs_addr dst, const float* src, unsigned bytes, rs_addr bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
// predicated forms (no branch: a lane-dependent branch in front of warp-wide shuffles leaves the warp diverged)
__device__ __forceinline__ void rs_bar_init_if(rs_addr bar, bool on) {
  asm volatile("{ .reg .pred p; setp.ne.b32 p, %1, 0; @p mbarrier.init.shared::cta.b64 [%0], 1; }" :: "r"(bar), "r"((int)on) : "memory");
}
__device__ __forceinline__ void rs_fetch_if(rs_addr dst, const float* src, unsigned bytes, rs_addr bar, bool on) {
  asm volatile("{ .reg .pred p; setp.ne.b32 p, %4, 0;\n"
               "  @p mbarrier.arrive.expect_tx.shared::cta.b64 _, [%3], %2;\n"
               "  @p cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3]; }"
               :: "r"(dst), "l"(src), "r"(bytes), "r"(bar), "r"((int)on) : "memory");
}
__device__ __forceinline__ bool rs_try_wait(rs_addr bar, unsigned parity) {
  unsigned ok;
  asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
               : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ void rs_wait(rs_addr bar, unsigned parity) {
  unsigned ok;
  do {
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  } while (!ok);
}
// The loop's per-entry arithmetic with its rounding pinned (explicit fma / mul / add, no contraction left to the
// compiler), so that the lane partition can change without changing a bit of the result:
//   J.v over the four blocks of one velocity entry: (j0 x0 + j1 x1) + (j2 x2 + j3 x3);
__device__ __forceinline__ float rs_jv(float j0, float x0, float j1, float x1, float j2, float x2, float j3, float x3) {
  return __fadd_rn(__fmaf_rn(j0, x0, __fmul_rn(j1, x1)), __fmaf_rn(j2, x2, __fmul_rn(j3, x3)));
}
//   the velocity update of one entry: x + m1 d1 + m2 d2.
__device__ __forceinline__ float rs_dv(float x, float m1, float d1, float m2, float d2) { return __fmaf_rn(m2, d2, __fmaf_rn(m1, d1, x)); }
struct RsHdr { v4 a, b, c, d; };
// 16-byte asynchronous copy global -> shared by the executing lane (LDGSTS), predicated, with a compile-time byte offset
template <int OFF> __device__ __forceinline__ void rs_cp16(rs_addr dst, const void* src, bool on) {
  asm volatile("{ .reg .pred p; setp.ne.b32 p, %2, 0; @p cp.async.cg.shared.global [%0+%3], [%1+%3], 16; }" :: "r"(dst), "l"(src), "r"((int)on), "n"(OFF) : "memory");
}
__device__ __forceinline__ void rs_cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int W> __device__ __forceinline__ void rs_cp_wait() { asm volatile("cp.async.wait_group %0;" :: "n"(W) : "memory"); }
// Shared-memory accesses of the K7 loop, as volatile asm on 32-bit shared addresses: they stay in program order (a
// velocity load must follow the previous record's store to the same entry) and never become generic loads.
__device__ __forceinline__ float rs_lds(rs_addr a) { float r; asm volatile("ld.shared.f32 %0, [%1];" : "=f"(r) : "r"(a)); return r; }
template <int OFF> __device__ __forceinline__ v4 rs_lds4(rs_addr a) {
  v4 r; asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4+%5];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "r"(a), "n"(OFF)); return r;
}
__device__ __forceinline__ float2 rs_lds2_if(rs_addr a, bool on) {         // zeros if not `on`
  float2 r; asm volatile("{ .reg .pred p; setp.ne.b32 p, %3, 0; mov.f32 %0, 0f00000000; mov.f32 %1, 0f00000000; @p ld.shared.v2.f32 {%0, %1}, [%2]; }"
                         : "=f"(r.x), "=f"(r.y) : "r"(a), "r"((int)on)); return r;
}
template <int OFF> __device__ __forceinline__ v4 rs_lds4_if(rs_addr a, bool on) {   // zeros if not `on`
  v4 r; asm volatile("{ .reg .pred p; setp.ne.b32 p, %5, 0; mov.f32 %0, 0f00000000; mov.f32 %1, 0f00000000; mov.f32 %2, 0f00000000; mov.f32 %3, 0f00000000;\n"
                     "  @p ld.shared.v4.f32 {%0, %1, %2, %3}, [%4+%6]; }" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "r"(a), "r"((int)on), "n"(OFF)); return r;
}
__device__ __forceinline__ void rs_sts(rs_addr a, float x) { asm volatile("st.shared.f32 [%0], %1;" :: "r"(a), "f"(x)); }
__device__ __forceinline__ void rs_sts2_if(rs_addr a, float x, float y, bool on) {
  asm volatile("{ .reg .pred p; setp.ne.b32 p, %3, 0; @p st.shared.v2.f32 [%0], {%1, %2}; }" :: "r"(a), "f"(x), "f"(y), "r"((int)on));
}
__device__ __forceinline__ void rs_sts4_if(rs_addr a, v4 x, bool on) {
  asm volatile("{ .reg .pred p; setp.ne.b32 p, %5, 0; @p st.shared.v4.f32 [%0], {%1, %2, %3, %4}; }" :: "r"(a), "f"(x.x), "f"(x.y), "f"(x.z), "f"(x.w), "r"((int)on));
}
__device__ __forceinline__ rs_addr rs_wrap(rs_addr ring, int byte) {        // ring | (byte & 4095): the ring is 4 KB aligned
  rs_addr r; asm("lop3.b32 %0, %1, 4095, %2, 0xEA;" : "=r"(r) : "r"(byte), "r"(ring)); return r;
}

#define RS_RING 1024          // floats of an env's stream ring (4 KB, 4 KB aligned)
#define RS_PIECE 32           // floats per refill piece: 4 lanes x 32 B
#define RS_KPF 6              // refill pieces per record consumed (192 floats > the largest record: the ring stays full)
#define RS_WAITG 3            // cp.async groups (= records) that may still be in flight

// One record of one env group.  (H, Q): header and lane blocks of the record solved now (loaded one trip earlier);
// (Hn, Qn): filled with the next record's.  Q[2k], Q[2k + 1]: quads 2l and 2l + 1 of lane block k.  See pgs_warp.
#define RS_TRIP(H, Q, Hn, Qn)                                                                                             \
  {                                                                                                                       \
    const int meta = f2i_bits(H.a.x), w1 = f2i_bits(H.a.y), w2 = f2i_bits(H.a.z), w3 = f2i_bits(H.a.w);                   \
    const int nv = meta & 7, mode = (meta >> 4) & 3;                                                                      \
    const rs_addr a0 = vbl + (w1 & 0xffff), a1 = vbl + ((unsigned)w1 >> 16), a2 = vbl + (w2 & 0xffff), a3 = vbl + ((unsigned)w2 >> 16); \
    const rs_addr l1 = vb + (w3 & 0xffff), l2 = vb + ((unsigned)w3 >> 16), ln = vb + f2i_bits(H.b.x);                     \
    const float2 x0 = rs_lds2_if(a0, nv > 0), x1 = rs_lds2_if(a1, nv > 1), x2 = rs_lds2_if(a2, nv > 2), x3 = rs_lds2_if(a3, nv > 3); \
    const float lam1 = rs_lds(l1), lam2 = rs_lds(l2), lamn = rs_lds(ln);                                                  \
    const int adv = active ? (int)((unsigned)meta >> 8) : 0;                                                              \
    const int nb = cb + adv;                                                                                              \
    left -= adv;                                                                                                          \
    const bool at_end = active && left == 0;                                                                              \
    left = at_end ? totalB : left;                                                                                        \
    rs_cp_wait<RS_WAITG>();                                                                                               \
    __syncwarp();                               /* pieces copied by the other lanes of the group */                       \
    const rs_addr ha = rs_wrap(ring_s, nb);                                                                               \
    Hn.a = rs_lds4<0>(ha); Hn.b = rs_lds4<16>(ha); Hn.c = rs_lds4<32>(ha); Hn.d = rs_lds4<48>(ha);                         \
    /* the partial sums of entries 2l and 2l + 1, added in a register: J.v is reduced over the same tree as with one */  \
    /* lane per entry (pairs, then xor 1 = pairs of pairs, then xor 2)                                                */  \
    float p1 = rs_jv(Q[0].x, x0.x, Q[2].x, x1.x, Q[4].x, x2.x, Q[6].x, x3.x) + rs_jv(Q[1].x, x0.y, Q[3].x, x1.y, Q[5].x, x2.y, Q[7].x, x3.y); \
    float p2 = rs_jv(Q[0].z, x0.x, Q[2].z, x1.x, Q[4].z, x2.x, Q[6].z, x3.x) + rs_jv(Q[1].z, x0.y, Q[3].z, x1.y, Q[5].z, x2.y, Q[7].z, x3.y); \
    p1 += __shfl_xor_sync(0xffffffffu, p1, 1); p2 += __shfl_xor_sync(0xffffffffu, p2, 1);                                 \
    /* refill: everything in front of the next record is consumed; up to RS_KPF pieces of 128 B right behind the */      \
    /* requests so far, not across the end of the ring or of the sweep (the next trip goes on from there)         */      \
    {                                                                                                                     \
      int n = min(min((nb + 4096 - pbyte) >> 7, (4096 - (pbyte & 4095)) >> 7), min((totalB - ppos) >> 7, RS_KPF));       \
      n = active ? n : 0;                                                                                                 \
      const rs_addr dst = rs_wrap(ring_s, pbyte) + 32 * l;                                                                \
      const char* src = rsl + ppos;                                                                                       \
      rs_cp16<0>(dst, src, n > 0); rs_cp16<16>(dst, src, n > 0); rs_cp16<128>(dst, src, n > 1); rs_cp16<144>(dst, src, n > 1); \
      rs_cp16<256>(dst, src, n > 2); rs_cp16<272>(dst, src, n > 2); rs_cp16<384>(dst, src, n > 3); rs_cp16<400>(dst, src, n > 3); \
      rs_cp16<512>(dst, src, n > 4); rs_cp16<528>(dst, src, n > 4); rs_cp16<640>(dst, src, n > 5); rs_cp16<656>(dst, src, n > 5); \
      rs_cp_commit();                                                                                                     \
      pbyte += n << 7; ppos += n << 7;                                                                                    \
      ppos = ppos == totalB ? 0 : ppos;                                                                                   \
    }                                                                                                                     \
    p1 += __shfl_xor_sync(0xffffffffu, p1, 2); p2 += __shfl_xor_sync(0xffffffffu, p2, 2);                                 \
    const RsSol r = rs_solve2(mode, cone_cfg, !active, p1, p2, lam1, lam2, lamn, H.c, H.d, H.b.y, H.b.z);                 \
    rs_sts(l1, r.s1); rs_sts(l2, r.s2);                                                                                   \
    rs_sts2_if(a0, rs_dv(x0.x, Q[0].y, r.d1, Q[0].w, r.d2), rs_dv(x0.y, Q[1].y, r.d1, Q[1].w, r.d2), nv > 0);             \
    rs_sts2_if(a1, rs_dv(x1.x, Q[2].y, r.d1, Q[2].w, r.d2), rs_dv(x1.y, Q[3].y, r.d1, Q[3].w, r.d2), nv > 1);             \
    rs_sts2_if(a2, rs_dv(x2.x, Q[4].y, r.d1, Q[4].w, r.d2), rs_dv(x2.y, Q[5].y, r.d1, Q[5].w, r.d2), nv > 2);             \
    rs_sts2_if(a3, rs_dv(x3.x, Q[6].y, r.d1, Q[6].w, r.d2), rs_dv(x3.y, Q[7].y, r.d1, Q[7].w, r.d2), nv > 3);             \
    resid = fmaxf(resid, fmaxf(r.d1 * r.d1, r.d2 * r.d2));                                                                \
    it += at_end ? 1 : 0;                                                                                                 \
    const bool stop = at_end && ((thr > 0.f && resid <= thr) || it >= iters);                                             \
    resid = at_end ? 0.f : resid;                                                                                         \
    /* a finished env parks: a null record (size 0) goes where its next record would have been read */                   \
    rs_sts4_if(ha + 16 * l, nullq, stop);                                                                                 \
    active = active && !stop;                                                                                             \
    cb = nb;                                                                                                              \
    /* lane blocks of the next record, last: its header has long arrived, so only its nv blocks are fetched; a lane's */ \
    /* two quads of a block are adjacent and never straddle the end of the ring                                        */ \
    {                                                                                                                     \
      const int nvn = f2i_bits(Hn.a.x) & 7;                                                                               \
      const int bl = nb + cl;                                                                                             \
      const rs_addr q0 = rs_wrap(ring_s, bl), q1 = rs_wrap(ring_s, bl + 128), q2 = rs_wrap(ring_s, bl + 256), q3 = rs_wrap(ring_s, bl + 384); \
      Qn[0] = rs_lds4_if<0>(q0, nvn > 0); Qn[1] = rs_lds4_if<16>(q0, nvn > 0);                                            \
      Qn[2] = rs_lds4_if<0>(q1, nvn > 1); Qn[3] = rs_lds4_if<16>(q1, nvn > 1);                                            \
      Qn[4] = rs_lds4_if<0>(q2, nvn > 2); Qn[5] = rs_lds4_if<16>(q2, nvn > 2);                                            \
      Qn[6] = rs_lds4_if<0>(q3, nvn > 3); Qn[7] = rs_lds4_if<16>(q3, nvn > 3);                                            \
    }                                                                                                                     \
  }

// One warp = eight envs (lane group g = lane / 4, lane l = lane % 4 of the group), lock-step.  Lane l owns entries 2l
// and 2l + 1 of every 8-entry velocity block (one LDS.64 / STS.64 per block) and quads 2l and 2l + 1 of every lane
// block (two LDS.128).  Shared memory: per env a 4 KB ring (4 KB aligned) through which the env's row stream flows
// once per sweep, then per env velocity deltas and impulses:
//   * the ring is filled by one TMA bulk copy per env (mbarrier complete_tx); a stream shorter than the ring wraps
//     inside it and is staged by cp.async pieces instead,
//   * from then on every lane copies its 32 B of each 128 B piece with two 16 B cp.async right behind the consumer (up
//     to RS_KPF pieces per record and env), so the refill is SIMT-uniform -- no elected lane, no spin loop -- and a
//     record is consumed RS_WAITG + 1 records after its bytes were requested (cp.async.wait_group).  Which bytes are
//     requested when does not depend on how the lanes split a piece: tests/test_ring_protocol.py models the schedule.
// The stream stays in HBM / L2; ~6.9 KB of shared memory per env keep every env of a 4096-env batch resident at once.
// There is NO lane-dependent branch in front of the loop's shuffles: a diverged warp executes them on a collective slow
// path that costs thousands of cycles per record (measured), so everything is selects and predicated instructions.
__device__ __forceinline__ void pgs_warp(const SimDev& S, float* sm, int, int warp_slot0) {
  const int lane = threadIdx.x & 31, g = lane >> 2, l = lane & 3;
  const int N = S.N;
  const int slot = warp_slot0 + g;
  const bool valid = slot < N;
  const int e = valid ? S.pgs_order[slot] : 0;
  const int NV = rs_nv(S), NL = rs_nlam(S), EF = NV + NL, ES = rs_env_stride(S);
  const rs_addr sm_s = rs_smem_addr(sm);
  const rs_addr ring0 = (sm_s + 4095u) & ~4095u;                    // the CTA asked for 4 KB of slack
  const rs_addr ring_s = ring0 + 4096u * g;
  float* v = (float*)((char*)sm + (ring0 - sm_s) + RS_CTA_ENVS * 4096) + (size_t)g * ES;
  const rs_addr vb = rs_smem_addr(v), vbl = vb + 8 * l;
  const rs_addr bar = rs_smem_addr(v - (size_t)g * ES + (size_t)RS_CTA_ENVS * ES) + 8 * g;
  const long long t_begin = clock64();
  for (int i = l; i < EF; i += 4) v[i] = 0.f;
  const float* rs = S.rs_data + (size_t)e * S.rs_cap;
  const char* rsl = (const char*)(rs + 8 * l);
  const int total = valid ? S.rs_nfloats[e] : 0;     // a multiple of RS_PIECE (K6a pads)
  const int totalB = total > 0 ? total * 4 : 128;
  v4 nullq;                                          // quad l of a null record's header
  nullq.x = rs_null_word(S, 4 * l); nullq.y = rs_null_word(S, 4 * l + 1); nullq.z = rs_null_word(S, 4 * l + 2); nullq.w = rs_null_word(S, 4 * l + 3);
  // ---- fill the ring (all of it: the stream repeats every sweep).  A stream of at least a ring: ONE TMA bulk copy;
  // a shorter one wraps inside the ring: 128 B pieces by cp.async; an env without rows: zeros and a null record.
  const bool big = total >= RS_RING;
  rs_bar_init_if(bar, l == 0);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncwarp();
  rs_fetch_if(ring_s, rs, RS_RING * 4, bar, l == 0 && big);
  {
    int pp = 0;
    v4 z; z.x = z.y = z.z = z.w = 0.f;
    for (int j = 0; j < RS_RING / RS_PIECE; j++) {
      rs_cp16<0>(ring_s + 128 * j + 32 * l, rsl + pp, !big && total > 0);
      rs_cp16<16>(ring_s + 128 * j + 32 * l, rsl + pp, !big && total > 0);
      rs_sts4_if(ring_s + 128 * j + 32 * l, z, total == 0);
      rs_sts4_if(ring_s + 128 * j + 32 * l + 16, z, total == 0);
      pp += 128; pp = pp >= totalB ? 0 : pp;
    }
    rs_cp_commit();
    rs_cp_wait<0>();
    __syncwarp();
    rs_sts4_if(ring_s + 16 * l, nullq, total == 0);
  }
  int ppos = (RS_RING * 4) % totalB, pbyte = RS_RING * 4;
  { bool ok; do { ok = big ? rs_try_wait(bar, 0) : true; } while (!__all_sync(0xffffffffu, ok)); }   // warp-uniform loop
  __syncwarp();
  bool active = total > 0 && S.iters > 0;
  int it = 0, cb = 0, left = totalB;
  const int cl = 64 + 32 * l;
  RsHdr HA, HB;
  v4 QA[8], QB[8];
  HA.a = rs_lds4<0>(ring_s); HA.b = rs_lds4<16>(ring_s); HA.c = rs_lds4<32>(ring_s); HA.d = rs_lds4<48>(ring_s);
  {
    const int nv0 = f2i_bits(HA.a.x) & 7;
    QA[0] = rs_lds4_if<0>(ring_s + cl, nv0 > 0); QA[1] = rs_lds4_if<16>(ring_s + cl, nv0 > 0);
    QA[2] = rs_lds4_if<128>(ring_s + cl, nv0 > 1); QA[3] = rs_lds4_if<144>(ring_s + cl, nv0 > 1);
    QA[4] = rs_lds4_if<256>(ring_s + cl, nv0 > 2); QA[5] = rs_lds4_if<272>(ring_s + cl, nv0 > 2);
    QA[6] = rs_lds4_if<384>(ring_s + cl, nv0 > 3); QA[7] = rs_lds4_if<400>(ring_s + cl, nv0 > 3);
  }
  HB = HA;
#pragma unroll
  for (int k = 0; k < 8; k++) QB[k] = QA[k];
  float resid = 0.f;
  const bool cone_cfg = S.cone != 0;
  const float thr = S.resid_thr;
  const int iters = S.iters;
  int guard = (S.iters * (S.rs_cap / RS_UNIT + 2) + 16) / 2 + 2;     // a corrupt stream must not hang the GPU
  const int guard0 = guard;
  bool act_lag = true;
  // The loop is software pipelined -- record t's header and lane blocks were loaded during record t-1 -- and unrolled
  // by two with the register sets swapped; the loop condition votes on the flag of two trips before (idle trips at the
  // end), so neither a load nor the vote sits on the dependent chain
  //   LDS v -> fma -> add -> 2 x (shfl, add) -> solve -> fma -> STS v.
  while (__any_sync(0xffffffffu, act_lag) && --guard > 0) {
    act_lag = active;
    RS_TRIP(HA, QA, HB, QB)
    RS_TRIP(HB, QB, HA, QA)
  }
  rs_cp_wait<0>();
  __syncwarp();
  if (!valid) return;
  // ---- write back and integrate (4 lanes per env): impulses for the read-back calls, then K8 straight from shared memory
  float* lam = v + NV;
  if (l == 0) { S.iters_used[e] = it; S.pgs_cycles[e] = (int)(clock64() - t_begin); S.pgs_trips[e] = 2 * (guard0 - guard); }
  const int ND = S.ND;
  for (int r = l; r < S.ngr; r += 4) S.gr_lam[(size_t)r * N + e] = lam[3 * ND + r];
  int cnt = S.c_count[e]; if (cnt > S.maxc) cnt = S.maxc;
  for (int i = l; i < 3 * cnt; i += 4) { int s = i / 3, c = i - 3 * s; cf_st(S.s_data, s, CF_LAM_N + c, N, e, lam[3 * ND + S.ngr + i]); }
  for (int d = l; d < ND; d += 4) {
    int k = AG_LDG(S.dl_link + d);
    if (S.body_mode[(size_t)AG_LDG(S.link_body + k) * N + e] == 1) st1(S.motor_applied, k, N, e, lam[2 * ND + d] / S.dt);
  }
  __syncwarp();                                    // c_count is clamped by lane 0 of the group in integrate_env
  struct DvShared { const float* v; const SimDev* S; __device__ __forceinline__ float operator()(int i) const {
    // entry i of the solver's velocity vector: dof d -> its articulation's block, free body f -> its 8-float block
    if (i >= S->ND) { int f = (i - S->ND) / 6, c = (i - S->ND) - 6 * f; return v[S->NDp + 8 * f + c]; }
    int a = AG_LDG(S->dl_art + i); return v[AG_LDG(S->art_voff + a) + (i - AG_LDG(S->art_dl0 + a))];
  } } dvs; dvs.v = v; dvs.S = &S;
  integrate_env(e, S, dvs, l, 4);
}
#endif

// Host restatement of the DEVICE loop of K7 for one env (tests only): the same ring indexing, refill schedule, software
// pipelining, finished-env parking and "blocks beyond nv are read but multiply zeros", with the asynchronous copies
// done synchronously.  It works entry by entry; how the device deals the entries to lanes (four lanes, two entries
// each) changes which lane computes what, not the byte schedule or the record order.  `sm`: rs_env_floats floats.
AG_HDN inline void pgs_env_emul(int slot, const SimDev& S, float* sm) {
  const int RING = 1024, KPF = 6;
  const int e = S.pgs_order[slot];
  const int N = S.N, ND = S.ND;
  const int NV = rs_nv(S), NL = rs_nlam(S);
  float* v = sm; float* lam = v + NV; float* ring = lam + NL + 64;
  for (int i = 0; i < NV + NL; i++) v[i] = 0.f;
  const float* rs = S.rs_data + (size_t)e * S.rs_cap;
  const int total = S.rs_nfloats[e];
  const int totalB = total > 0 ? total * 4 : 128;
  for (int i = 0; i < RING; i++) ring[i] = total > 0 ? rs[i % total] : 0.f;
  if (total == 0) for (int i = 0; i < 16; i++) ring[i] = rs_null_word(S, i);
  int ppos = (RING * 4) % totalB, pbyte = RING * 4;
  bool active = total > 0 && S.iters > 0;
  int it = 0, cb = 0, left = totalB;
  float H[16], Q[4][8][4];
  for (int i = 0; i < 16; i++) H[i] = ring[i];
  for (int k = 0; k < 4; k++) for (int l = 0; l < 8; l++) for (int c = 0; c < 4; c++) Q[k][l][c] = ring[RS_HDR + k * RS_LB + 4 * l + c];
  float resid = 0.f;
  bool act_lag = true;
  long guard = (long)S.iters * (S.rs_cap / RS_UNIT + 2) + 16;
  for (int half = 0; (half & 1) || (act_lag && --guard > 0); half++) {
    if (!(half & 1)) act_lag = active;                    // the device loop votes once per two trips
    const int meta = f2i_bits(H[0]), w1 = f2i_bits(H[1]), w2 = f2i_bits(H[2]), w3 = f2i_bits(H[3]);
    const int nv = meta & 7, mode = (meta >> 4) & 3;
    const int sl[4] = {(w1 & 0xffff) / 4, (int)((unsigned)w1 >> 16) / 4, (w2 & 0xffff) / 4, (int)((unsigned)w2 >> 16) / 4};
    float* lp1 = v + (w3 & 0xffff) / 4; float* lp2 = v + ((unsigned)w3 >> 16) / 4;
    const float lam1 = *lp1, lam2 = *lp2, lamn = v[f2i_bits(H[4]) / 4];
    const int adv = active ? (int)((unsigned)meta >> 8) : 0;
    const int nb = cb + adv;
    left -= adv;
    const bool at_end = active && left == 0;
    left = at_end ? totalB : left;
    float Hn[16], Qn[4][8][4];
    for (int i = 0; i < 16; i++) Hn[i] = ring[((nb / 4) + i) & (RING - 1)];
    for (int k = 0; k < 4; k++) for (int l = 0; l < 8; l++) for (int c = 0; c < 4; c++) Qn[k][l][c] = ring[((nb / 4) + RS_HDR + k * RS_LB + 4 * l + c) & (RING - 1)];
    float p1 = 0.f, p2 = 0.f, x[4][8];
    for (int l = 0; l < 8; l++) { for (int k = 0; k < 4; k++) x[k][l] = v[sl[k] + l];
      p1 += (Q[0][l][0] * x[0][l] + Q[1][l][0] * x[1][l]) + (Q[2][l][0] * x[2][l] + Q[3][l][0] * x[3][l]);
      p2 += (Q[0][l][2] * x[0][l] + Q[1][l][2] * x[1][l]) + (Q[2][l][2] * x[2][l] + Q[3][l][2] * x[3][l]); }
    {
      int n = (nb + 4096 - pbyte) >> 7;
      if (((4096 - (pbyte & 4095)) >> 7) < n) n = (4096 - (pbyte & 4095)) >> 7;
      if (((totalB - ppos) >> 7) < n) n = (totalB - ppos) >> 7;
      if (n > KPF) n = KPF;
      if (!active) n = 0;
      for (int i = 0; i < 32 * n; i++) ring[((pbyte / 4) + i) & (RING - 1)] = rs[ppos / 4 + i];
      pbyte += n << 7; ppos += n << 7;
      ppos = ppos == totalB ? 0 : ppos;
    }
    v4 hc, hd; hc.x = H[8]; hc.y = H[9]; hc.z = H[10]; hc.w = H[11]; hd.x = H[12]; hd.y = H[13]; hd.z = H[14]; hd.w = H[15];
    const RsSol r = rs_solve2(mode, S.cone != 0, !active, p1, p2, lam1, lam2, lamn, hc, hd, H[5], H[6]);
    *lp1 = r.s1; *lp2 = r.s2;
    for (int k = 0; k < nv; k++) for (int l = 0; l < 8; l++) v[sl[k] + l] = x[k][l] + Q[k][l][1] * r.d1 + Q[k][l][3] * r.d2;
    resid = fmaxf(resid, fmaxf(r.d1 * r.d1, r.d2 * r.d2));
    it += at_end ? 1 : 0;
    const bool stop = at_end && ((S.resid_thr > 0.f && resid <= S.resid_thr) || it >= S.iters);
    resid = at_end ? 0.f : resid;
    if (stop) for (int i = 0; i < 16; i++) ring[((nb / 4) + i) & (RING - 1)] = rs_null_word(S, i);
    active = active && !stop;
    cb = nb;
    for (int i = 0; i < 16; i++) H[i] = Hn[i];
    memcpy(Q, Qn, sizeof(Q));
  }
  S.iters_used[e] = it;
  for (int a = 0; a < S.nart; a++) {
    int d0 = AG_LDG(S.art_dl0 + a), nd = AG_LDG(S.art_nd + a), vo = AG_LDG(S.art_voff + a);
    for (int i = 0; i < nd; i++) S.dv[(size_t)(d0 + i) * N + e] = v[vo + i];
  }
  for (int f = 0; f < S.nf; f++)
    for (int c = 0; c < 6; c++) S.dv[(size_t)(ND + 6 * f + c) * N + e] = v[S.NDp + 8 * f + c];
  for (int r = 0; r < 3 * ND; r++) S.dr_lam[(size_t)r * N + e] = lam[r];
  for (int r = 0; r < S.ngr; r++) S.gr_lam[(size_t)r * N + e] = lam[3 * ND + r];
  int cnt = S.c_count[e]; if (cnt > S.maxc) cnt = S.maxc;
  for (int s2 = 0; s2 < cnt; s2++) {
    const float* ll = lam + 3 * ND + S.ngr + 3 * s2;
    cf_st(S.s_data, s2, CF_LAM_N, N, e, ll[0]);
    cf_st(S.s_data, s2, CF_LAM_T1, N, e, ll[1]);
    cf_st(S.s_data, s2, CF_LAM_T2, N, e, ll[2]);
  }
}

// Host restatement of K7 for the kernel-logic harness (tests only): the same stream, records consumed one after the
// other, entries summed in lane-block order.  `sm`: rs_nv + rs_nlam floats.
AG_HDN inline void pgs_body_host(int slot, const SimDev& S, float* sm) {
  const int e = S.pgs_order[slot];
  const int N = S.N, ND = S.ND;
  const int NV = rs_nv(S), NL = rs_nlam(S);
  float* v = sm; float* lam = sm + NV;
  for (int i = 0; i < NV + NL; i++) sm[i] = 0.f;
  const float* rs = S.rs_data + (size_t)e * S.rs_cap;
  const int total = S.rs_nfloats[e];
  int used = 0;
  for (int it = 0; it < S.iters && total > 0; it++) {
    float resid = 0.f;
    used = it + 1;
    for (int pos = 0; pos < total;) {
      const float* rec = rs + pos;
      const int meta = f2i_bits(rec[0]), w1 = f2i_bits(rec[1]), w2 = f2i_bits(rec[2]), w3 = f2i_bits(rec[3]);
      const int nv = meta & 7, mode = (meta >> 4) & 3, size = rs_meta_floats(meta);
      pos += size > 0 ? size : RS_UNIT;
      if (mode == RM_PAD) continue;
      const int sl[4] = {(w1 & 0xffff) / 4, (w1 >> 16) / 4, (w2 & 0xffff) / 4, (w2 >> 16) / 4};
      float p1 = 0.f, p2 = 0.f;
      for (int kk = 0; kk < nv; kk++) for (int l = 0; l < 8; l++) { const float* q = rec + RS_HDR + kk * RS_LB + 4 * l; float x = v[sl[kk] + l]; p1 += q[0] * x; p2 += q[2] * x; }
      float* lp1 = v + (w3 & 0xffff) / 4; float* lp2 = v + (w3 >> 16) / 4;
      RsSol r = rs_solve2(mode, S.cone != 0, false, p1, p2, *lp1, *lp2, v[f2i_bits(rec[4]) / 4], ldv4(rec + 8), ldv4(rec + 12), rec[5], rec[6]);
      *lp1 = r.s1; *lp2 = r.s2;
      for (int kk = 0; kk < nv; kk++) for (int l = 0; l < 8; l++) { const float* q = rec + RS_HDR + kk * RS_LB + 4 * l; v[sl[kk] + l] += q[1] * r.d1 + q[3] * r.d2; }
      resid = fmaxf(resid, fmaxf(r.d1 * r.d1, r.d2 * r.d2));
    }
    if (S.resid_thr > 0.f && resid <= S.resid_thr) break;
  }
  S.iters_used[e] = used;
  for (int a = 0; a < S.nart; a++) {
    int d0 = AG_LDG(S.art_dl0 + a), nd = AG_LDG(S.art_nd + a), vo = AG_LDG(S.art_voff + a);
    for (int i = 0; i < nd; i++) S.dv[(size_t)(d0 + i) * N + e] = v[vo + i];
  }
  for (int f = 0; f < S.nf; f++)
    for (int c = 0; c < 6; c++) S.dv[(size_t)(ND + 6 * f + c) * N + e] = v[S.NDp + 8 * f + c];
  for (int r = 0; r < 3 * ND; r++) S.dr_lam[(size_t)r * N + e] = lam[r];
  for (int r = 0; r < S.ngr; r++) S.gr_lam[(size_t)r * N + e] = lam[3 * ND + r];
  int cnt = S.c_count[e]; if (cnt > S.maxc) cnt = S.maxc;
  for (int s = 0; s < cnt; s++) {
    const float* ll = lam + 3 * ND + S.ngr + 3 * s;
    cf_st(S.s_data, s, CF_LAM_N, N, e, ll[0]);
    cf_st(S.s_data, s, CF_LAM_T1, N, e, ll[1]);
    cf_st(S.s_data, s, CF_LAM_T2, N, e, ll[2]);
  }
}
