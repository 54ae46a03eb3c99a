// TEST INFRASTRUCTURE ONLY: sequential host driver for the frame functions of glamr_b200/csrc/globalopt_frames.cuh on a problem of
// G seed groups (include/glamr_b200.h, glamr_problem_t.G).  Same kernel sequence as emu.cpp, with every per-frame camera step run
// over the G*T camera rows and the term sums kept per group, so tests/test_seed_batch.py can hold a two-group problem to two
// one-group problems term by term and gradient by gradient.  Never used by the product.
#include <math.h>
#include <string.h>

#include <vector>

#include "../../glamr_b200/csrc/globalopt_frames.cuh"

using namespace glamr;

struct GroupEmu {
  glamr_problem_t pb;
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

static OptCtx make_ctx(GroupEmu* h, const float* theta, float* grad) {
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

int glamr_group_emu_create(GroupEmu** out, const glamr_problem_t* pb) {
  GroupEmu* h = new GroupEmu();
  h->pb = *pb;
  const size_t N = (size_t)pb->P * pb->T, GT = (size_t)num_groups(*pb) * pb->T, J = pb->J;
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
int glamr_group_emu_destroy(GroupEmu* h) { delete h; return 0; }

// trajectory + camera forward of every person and camera row
int glamr_group_emu_forward_pose(GroupEmu* h, const float* theta) {
  OptCtx c = make_ctx(h, theta, nullptr);
  const glamr_problem_t& pb = h->pb;
  for (int p = 0; p < pb.P; ++p) {
    const glamr_person_t& ps = pb.persons[p];
    const size_t n0 = (size_t)p * pb.T + ps.start;
    for (int i = 0; i < ps.len; ++i) traj_pre(c, p, i);
    scan(c.sc.heading + n0, ps.len, 1, false);
    for (int i = 0; i < ps.len; ++i) traj_mid(c, p, i);
    scan(c.sc.xy + 2 * n0, ps.len, 2, false);
    scan(c.sc.xy + 2 * n0 + 1, ps.len, 2, false);
    for (int t = 0; t < pb.T; ++t) traj_post(c, p, t);
  }
  for (int gt = 0; gt < num_groups(pb) * pb.T; ++gt) cam_forward(c, gt);
  return 0;
}

// what: 0 orient_world [P,T,3], 1 trans_world, 2 joints_world [P,T,J,3] (filled by the caller), 3 cam [G,T,12]
int glamr_group_emu_buffer(GroupEmu* h, int what, float** ptr, size_t* count) {
  const size_t N = (size_t)h->pb.P * h->pb.T, GT = (size_t)num_groups(h->pb) * h->pb.T, J = h->pb.J;
  switch (what) {
    case 0: *ptr = h->sc.orient_world; *count = 3 * N; break;
    case 1: *ptr = h->sc.trans_world; *count = 3 * N; break;
    case 2: *ptr = h->sc.joints_world; *count = N * J * 3; break;
    case 3: *ptr = h->sc.cam; *count = 12 * GT; break;
    default: return -1;
  }
  return 0;
}

// residuals + backward: reduce_buf = [grad | G x term sums]; each group's terms are summed in the order of its one-group problem
int glamr_group_emu_backward(GroupEmu* h, const float* theta, float* reduce_buf) {
  const glamr_problem_t& pb = h->pb;
  const int G = num_groups(pb), Q = group_persons(pb), T = pb.T;
  memset(reduce_buf, 0, sizeof(float) * ((size_t)pb.n_params + (size_t)G * GLAMR_NUM_TERMS));
  OptCtx c = make_ctx(h, theta, reduce_buf);
  std::vector<TermAcc> acc(G);
  for (int g = 0; g < G; ++g) acc[g].clear();
  for (int p = 0; p < pb.P; ++p)
    for (int t = 0; t < T; ++t) frame_residuals(c, p, t, acc[p / Q]);
  for (int gt = 0; gt < G * T; ++gt) camera_backward(c, gt, acc[gt / T]);
  if (pb.cam_mode == GLAMR_CAM_FROM_PERSONS)
    for (int gs = 0; gs < G * T; ++gs) camera_scatter_to_persons(c, gs);
  for (int p = 0; p < pb.P; ++p) {
    const glamr_person_t& ps = pb.persons[p];
    const size_t n0 = (size_t)p * T + ps.start;
    TermAcc& a = acc[p / Q];
    for (int t = 0; t < T; ++t) traj_back_pre(c, p, t, a);
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
      for (int t = 0; t < T; ++t)
        for (int k = 0; k < 9; ++k) a[k] += c.sc.g_cam_fix[((size_t)g * T + t) * 12 + k];
      for (int k = 0; k < 9; ++k)
        reduce_buf[group_theta(pb, g) + ((k < 6) ? pb.off_cam_rot + k : pb.off_cam_trans + (k - 6))] = (float)a[k];
    }
  }
  return 0;
}
}
