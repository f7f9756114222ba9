// schedule.cu -- a device-resident view schedule (gab200_schedule_sample / gab200_schedule_commit): each replay of a
// captured frame picks its own record, so a run of replays takes no host input.
//
// The schedule is a table of R records -- K camera rows of 37 floats, a FLAME timestep and K frame ids each -- and an
// order of L record indices.  A device cursor c names the iteration.  The sampler, at the head of the replay, copies
// record order[c] into the frame's static inputs; the commit, at its end, advances the cursor unless the replay
// overflowed its instance capacity (the slot's sticky flag) or found the schedule exhausted.  So an overflowed replay
// and every replay after it in the same run leave the cursor where it was, and the run resumes at that record.
//
// Both are plain launches (no programmatic dependent launch): the sampler completes before the next kernel starts,
// and that kernel (the FLAME pose, a plain launch, or a launch_pdl kernel that reads the camera below pdl_wait())
// sees its writes.
#include "common.cuh"
#include "kernels.cuh"

namespace gab {

namespace {

constexpr int SCHED_THREADS = 256;

// One CTA.  c = *cursor; c outside [0, length) or a record index outside [0, records): write nothing but *exhausted.
__global__ void __launch_bounds__(SCHED_THREADS) schedule_sample_kernel(
    int records, int views, int length, const float* __restrict__ cams, const int32_t* __restrict__ timesteps,
    const int32_t* __restrict__ frame_ids, const int32_t* __restrict__ order, const int32_t* __restrict__ cursor,
    float* __restrict__ cam_out, int32_t* __restrict__ timestep_out, int32_t* __restrict__ ids_out,
    int32_t* __restrict__ rows_out, int32_t* __restrict__ exhausted) {
  const int c = *cursor;
  const int r = (c >= 0 && c < length) ? order[c] : -1;
  if (r < 0 || r >= records) {
    if (threadIdx.x == 0) *exhausted = 1;
    return;
  }
  const int64_t n = (int64_t)views * GAB200_CAMERA_FLOATS;
  const float* src = cams + (int64_t)r * n;
  for (int64_t i = threadIdx.x; i < n; i += SCHED_THREADS) cam_out[i] = src[i];
  for (int k = threadIdx.x; k < views; k += SCHED_THREADS) {
    const int64_t row = (int64_t)r * views + k;
    if (ids_out != nullptr) ids_out[k] = frame_ids[row];
    if (rows_out != nullptr) rows_out[k] = (int32_t)row;
  }
  if (threadIdx.x == 0 && timestep_out != nullptr) *timestep_out = timesteps[r];
}

// One thread: the replay's record is done unless it overflowed or the schedule was exhausted.
__global__ void schedule_commit_kernel(int length, const int32_t* __restrict__ overflow_flag,
                                       const int32_t* __restrict__ exhausted, const float* __restrict__ loss,
                                       float* __restrict__ losses, int32_t* __restrict__ cursor) {
  if ((overflow_flag != nullptr && *overflow_flag != 0) || *exhausted != 0) return;
  const int c = *cursor;
  if (c < 0 || c >= length) return;
  if (losses != nullptr) losses[c] = *loss;
  *cursor = c + 1;
}

}  // namespace

void launch_schedule_sample(int records, int views, int length, const float* cams, const int32_t* timesteps,
                            const int32_t* frame_ids, const int32_t* order, const int32_t* cursor, float* cam_out,
                            int32_t* timestep_out, int32_t* ids_out, int32_t* rows_out, int32_t* exhausted,
                            cudaStream_t stream) {
  schedule_sample_kernel<<<1, SCHED_THREADS, 0, stream>>>(records, views, length, cams, timesteps, frame_ids, order,
                                                          cursor, cam_out, timestep_out, ids_out, rows_out, exhausted);
  count_launch();
}

void launch_schedule_commit(int length, const int32_t* overflow_flag, const int32_t* exhausted, const float* loss,
                            float* losses, int32_t* cursor, cudaStream_t stream) {
  schedule_commit_kernel<<<1, 1, 0, stream>>>(length, overflow_flag, exhausted, loss, losses, cursor);
  count_launch();
}

}  // namespace gab
