// TEST INFRASTRUCTURE ONLY: sequential host driver for the frame functions of glamr_b200/csrc/globalopt_frames.cuh on a problem of
// groups that differ in frames, persons, gaps and normalisers (include/glamr_b200.h, glamr_group_t).  Same kernel sequence as
// emu_groups.cpp, with every index taken from the group table: each person's rows start at its group's first frame-person, each
// group's camera rows at its first camera row, and the term sums are kept per group.  tests/test_sequence_batch.py holds such a
// problem to its one-group problems term by term and gradient by gradient.  Never used by the product.
#include <math.h>
#include <string.h>

#include <vector>

#include "../../glamr_b200/csrc/globalopt_frames.cuh"

using namespace glamr;

struct BatchEmu {
  glamr_problem_t pb;
  size_t N, rows;
  std::vector<float> buf[24];
  OptScratch sc;
};

static void scan(float* d, int count, int stride, bool reverse) {
  float run = 0.0f;
  for (int k = 0; k < count; ++k) {
    const int idx = reverse ? count - 1 - k : k;
    run += d[(size_t)idx * stride];
    d[(size_t)idx * stride] = run;
  }
}

static OptCtx make_ctx(BatchEmu* h, const float* theta, float* grad) {
  OptCtx c;
  c.pb = h->pb;
  c.sc = h->sc;
  c.sc.grad = grad;
  c.theta = theta;
  for (int k = 0; k < GLAMR_NUM_TERMS; ++k) {
    const glamr_problem_t& pb = h->pb;
    c.gs[k] = (pb.term_enabled[k] && !pb.term_monitor[k] && pb.term_norm[k] != 0.0f) ? pb.term_weight[k] / pb.term_norm[k] : 0.0f;
  }
  return c;
}

extern "C" {

int glamr_batch_emu_create(BatchEmu** out, const glamr_problem_t* pb) {
  BatchEmu* h = new BatchEmu();
  h->pb = *pb;
  h->N = 0;
  h->rows = 0;
  for (int g = 0; g < num_groups(*pb); ++g) {
    h->N += (size_t)group_persons(*pb, g) * group_frames(*pb, g);
    h->rows += group_frames(*pb, g);
  }
  const size_t N = h->N, GT = h->rows, J = pb->J;
  int i = 0;
  auto take = [&](size_t n) { h->buf[i].assign(n, 0.0f); return h->buf[i++].data(); };
  h->sc.heading = take(N); h->sc.xy = take(2 * N); h->sc.traj_local = take(11 * N); h->sc.orient_base = take(3 * N);
  h->sc.trans_base = take(3 * N); h->sc.orient_world = take(3 * N); h->sc.trans_world = take(3 * N); h->sc.cam = take(12 * GT);
  h->sc.cam_inv = take(12 * GT); h->sc.cam_d6 = take(6 * GT); h->sc.joints_world = take(N * J * 3); h->sc.kp_pred = take(N * J * 2);
  h->sc.orient_ciw = take(3 * N); h->sc.trans_ciw = take(3 * N); h->sc.g_orient = take(3 * N); h->sc.g_trans = take(3 * N);
  h->sc.g_cam = take(12 * N); h->sc.g_cam_fix = take(12 * GT); h->sc.g_xy = take(2 * N); h->sc.g_head = take(N);
  h->sc.grad = nullptr;
  *out = h;
  return 0;
}
int glamr_batch_emu_destroy(BatchEmu* h) { delete h; return 0; }

// trajectory + camera forward of every person and camera row
int glamr_batch_emu_forward_pose(BatchEmu* h, const float* theta) {
  OptCtx c = make_ctx(h, theta, nullptr);
  const glamr_problem_t& pb = h->pb;
  for (int p = 0; p < pb.P; ++p) {
    const glamr_person_t& ps = pb.persons[p];
    const size_t n0 = person_row(pb, p) + ps.start;
    for (int i = 0; i < ps.len; ++i) traj_pre(c, p, i);
    scan(c.sc.heading + n0, ps.len, 1, false);
    for (int i = 0; i < ps.len; ++i) traj_mid(c, p, i);
    scan(c.sc.xy + 2 * n0, ps.len, 2, false);
    scan(c.sc.xy + 2 * n0 + 1, ps.len, 2, false);
    for (int t = 0; t < person_frames(pb, p); ++t) traj_post(c, p, t);
  }
  for (int r = 0; r < (int)h->rows; ++r) cam_forward(c, r);
  return 0;
}

// what: 0 orient_world [N,3], 1 trans_world, 2 joints_world [N,J,3] (filled by the caller), 3 cam [sum T,12]
int glamr_batch_emu_buffer(BatchEmu* h, int what, float** ptr, size_t* count) {
  const size_t N = h->N, J = h->pb.J;
  switch (what) {
    case 0: *ptr = h->sc.orient_world; *count = 3 * N; break;
    case 1: *ptr = h->sc.trans_world; *count = 3 * N; break;
    case 2: *ptr = h->sc.joints_world; *count = N * J * 3; break;
    case 3: *ptr = h->sc.cam; *count = 12 * h->rows; break;
    default: return -1;
  }
  return 0;
}

// residuals + backward: reduce_buf = [grad | G x term sums]; each group's terms are summed in the order of its one-group problem
int glamr_batch_emu_backward(BatchEmu* h, const float* theta, float* reduce_buf) {
  const glamr_problem_t& pb = h->pb;
  const int G = num_groups(pb);
  memset(reduce_buf, 0, sizeof(float) * ((size_t)pb.n_params + (size_t)G * GLAMR_NUM_TERMS));
  OptCtx c = make_ctx(h, theta, reduce_buf);
  std::vector<TermAcc> acc(G);
  for (int g = 0; g < G; ++g) acc[g].clear();
  for (int p = 0; p < pb.P; ++p)
    for (int t = 0; t < person_frames(pb, p); ++t) frame_residuals(c, p, t, acc[person_group(pb, p)]);
  for (int r = 0; r < (int)h->rows; ++r) camera_backward(c, r, acc[cam_row_group(pb, r)]);
  if (pb.cam_mode == GLAMR_CAM_FROM_PERSONS)
    for (int r = 0; r < (int)h->rows; ++r) camera_scatter_to_persons(c, r);
  for (int p = 0; p < pb.P; ++p) {
    const glamr_person_t& ps = pb.persons[p];
    const size_t n0 = person_row(pb, p) + ps.start;
    TermAcc& a = acc[person_group(pb, p)];
    for (int t = 0; t < person_frames(pb, p); ++t) traj_back_pre(c, p, t, a);
    scan(c.sc.g_xy + 2 * n0, ps.len, 2, true);
    scan(c.sc.g_xy + 2 * n0 + 1, ps.len, 2, true);
    for (int i = 0; i < ps.len; ++i) traj_back_mid(c, p, i, a);
    scan(c.sc.g_head + n0, ps.len, 1, true);
    for (int i = 0; i < ps.len; ++i) traj_back_post(c, p, i, a);
  }
  for (int g = 0; g < G; ++g)
    for (int k = 0; k < GLAMR_NUM_TERMS; ++k) reduce_buf[pb.n_params + g * GLAMR_NUM_TERMS + k] = (float)acc[g].v[k];
  if (pb.cam_mode == GLAMR_CAM_FIXED) {
    for (int g = 0; g < G; ++g) {
      double a[9] = {0};
      const size_t r0 = group_cam_row0(pb, g);
      for (int t = 0; t < group_frames(pb, g); ++t)
        for (int k = 0; k < 9; ++k) a[k] += c.sc.g_cam_fix[(r0 + t) * 12 + k];
      for (int k = 0; k < 9; ++k)
        reduce_buf[(k < 6) ? group_off_cam_rot(pb, g) + k : group_off_cam_trans(pb, g) + (k - 6)] = (float)a[k];
    }
  }
  return 0;
}
}
