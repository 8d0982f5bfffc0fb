// yolov3_b200 — whole-graph executor: an immutable list of prepared launches (TMA descriptors encoded once) that
// replays Model.forward (reference models/yolo.py:135-147 _forward_once + Detect) on one stream with no host work
// between kernels beyond the launches themselves; capturable into a CUDA graph by the caller.
#include <new>
#include <vector>

#include "y3_internal.h"

struct y3_model {
  struct Step {
    int kind;
    y3::ConvTcPlan conv;
    y3_first_desc first;
    y3_pool_desc pool;
    y3_decode_desc decode;
    y3_amax_desc amax;
  };
  std::vector<Step> steps;
};

extern "C" int y3_model_create(const y3_op* ops, int32_t n_ops, y3_model** out) {
  Y3_REQUIRE(ops && out && n_ops > 0, "model_create: bad arguments");
  int rc = y3_device_check();
  if (rc) return rc;
  y3_model* m = new (std::nothrow) y3_model();
  if (!m) return y3::set_error(Y3_ERR_BAD_ARG, "model_create: out of host memory");
  m->steps.resize(n_ops);
  for (int i = 0; i < n_ops; ++i) {
    y3_model::Step& s = m->steps[i];
    s.kind = ops[i].kind;
    switch (ops[i].kind) {
      case Y3_OP_CONV:
        rc = y3::conv_tc_prepare(ops[i].conv, &s.conv);
        break;
      case Y3_OP_CONV_FIRST:
        s.first = ops[i].first;
        break;
      case Y3_OP_MAXPOOL:
        s.pool = ops[i].pool;
        break;
      case Y3_OP_DECODE:
        s.decode = ops[i].decode;
        break;
      case Y3_OP_AMAX:
        s.amax = ops[i].amax;
        break;
      default:
        rc = y3::set_error(Y3_ERR_BAD_ARG, "model_create: op %d has unknown kind %d", i, ops[i].kind);
    }
    if (rc) {
      char buf[400];
      y3_last_error(buf, sizeof(buf));
      delete m;
      return y3::set_error(rc, "model_create: op %d: %s", i, buf);
    }
  }
  *out = m;
  return Y3_OK;
}

static int launch_step(const y3_model::Step& s, const void* input, y3_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  switch (s.kind) {
    case Y3_OP_CONV:
      return y3::conv_tc_launch(s.conv, stream);
    case Y3_OP_CONV_FIRST: {
      y3_first_desc f = s.first;
      if (input) f.in = input;
      return y3_conv_first_fwd(&f, stream_);
    }
    case Y3_OP_MAXPOOL:
      return y3::pool_launch(s.pool, stream);
    case Y3_OP_DECODE:
      return y3_detect_head_decode_fwd(&s.decode, stream_);
    case Y3_OP_AMAX:
      return y3::amax_launch(s.amax, stream);
  }
  return Y3_OK;
}

// Profiling aid (NOT graph capturable, synchronises): per-launch device time via CUDA events on `stream`.
extern "C" int y3_model_forward_timed(const y3_model* m, const void* input, y3_stream_t stream_, float* ms_out,
                                      int32_t iters) {
  Y3_REQUIRE(m && ms_out && iters > 0, "model_forward_timed: bad arguments");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const size_t n = m->steps.size();
  std::vector<cudaEvent_t> ev(n + 1);
  for (auto& e : ev) Y3_CHECK_CUDA(cudaEventCreate(&e));
  for (size_t i = 0; i < n; ++i) ms_out[i] = 0.f;
  int rc = Y3_OK;
  for (int it = 0; it < iters && rc == Y3_OK; ++it) {
    Y3_CHECK_CUDA(cudaEventRecord(ev[0], stream));
    for (size_t i = 0; i < n && rc == Y3_OK; ++i) {
      rc = launch_step(m->steps[i], input, stream_);
      if (rc == Y3_OK && cudaEventRecord(ev[i + 1], stream) != cudaSuccess) rc = Y3_ERR_CUDA;
    }
    if (rc == Y3_OK && cudaStreamSynchronize(stream) != cudaSuccess) rc = y3::set_error(Y3_ERR_CUDA, "sync failed");
    for (size_t i = 0; i < n && rc == Y3_OK; ++i) {
      float ms = 0.f;
      cudaEventElapsedTime(&ms, ev[i], ev[i + 1]);
      ms_out[i] += ms / iters;
    }
  }
  for (auto& e : ev) cudaEventDestroy(e);
  return rc;
}

extern "C" int y3_model_forward(const y3_model* m, const void* input, y3_stream_t stream_) {
  Y3_REQUIRE(m, "model_forward: null model");
  for (size_t i = 0; i < m->steps.size(); ++i) {
    const int rc = launch_step(m->steps[i], input, stream_);
    if (rc) return rc;
  }
  return Y3_OK;
}

extern "C" int32_t y3_model_num_launches(const y3_model* m) { return m ? static_cast<int32_t>(m->steps.size()) : 0; }

extern "C" void y3_model_destroy(y3_model* m) { delete m; }
