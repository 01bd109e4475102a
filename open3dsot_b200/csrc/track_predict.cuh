// The centre a live-tracker row writes on an advance before any detection is taken into account: the network's box P on a hit
// (or without the end-of-track rule), the coasted centre hit_c + vel * gap on a miss under coasting.  Shared by the write-back
// (track_update.cu), which writes it, and the detection matching (associate.cu), which matches detections against it, so that
// both compute it with the same rounded fp32 operations (tracking/multi_tracker.py track_update_tensors / associate_tensors).
#pragma once

// gap = (float)(t' - hit_t), t' the row's frame counter after this advance
__device__ __forceinline__ void o3d_predicted_centre(const float pc[3], bool hit, bool coast, const float hit_c[3],
                                                     const float vel[3], float gap, float out[3]) {
#pragma unroll
    for (int j = 0; j < 3; ++j) out[j] = (coast && !hit) ? __fadd_rn(hit_c[j], __fmul_rn(vel[j], gap)) : pc[j];
}
