/* oracle/blend_oracle.c -- TEST INFRASTRUCTURE ONLY: the port's rtm::qvv_lerp over a pose as an entry point of its own, built into
 * liboracle_blend.so by oracle/blend.mk. The restatements it needs (dot_bias_dpps, metric_quat_normalize, lerpf) are file-local to
 * acl_oracle.c, so that file is compiled in here unchanged. */
#include "acl_oracle.c"

/* rtm::qvv_lerp(from, to, weight), qvvf.h:439-445, on every bone of one pose of rtm::qvvf rows (12 floats): quat_lerp's SSE4.1 path
 * (quatf.h:1006-1075: the sign bit of the dpps dot flips `to`, (s - w s) + w (e ^ bias)) normalised in `normalize_mode` (0: rsqrtss + 2
 * Newton-Raphson steps as the reference, 1: IEEE 1 / sqrt as the CUDA path), vector_lerp (vector4f.h:2417-2421) for translation and scale.
 * The translation and scale w lanes are written as 0. */
void aclo_qvv_lerp(const float* from_pose, const float* to_pose, uint32_t num_tracks, float weight, int normalize_mode, float* out_pose)
{
	for (uint32_t bone = 0; bone < num_tracks; ++bone)
	{
		const float* s = from_pose + (size_t)bone * 12;
		const float* e = to_pose + (size_t)bone * 12;
		float out[12];
		const uint32_t bias = dot_bias_dpps(s, e);
		for (int i = 0; i < 4; ++i)
			out[i] = (s[i] - weight * s[i]) + weight * u32_as_f32(f32_as_u32(e[i]) ^ bias);
		metric_quat_normalize(out, normalize_mode);
		for (int i = 0; i < 3; ++i)
		{
			out[4 + i] = lerpf(s[4 + i], e[4 + i], weight);
			out[8 + i] = lerpf(s[8 + i], e[8 + i], weight);
		}
		out[7] = 0.0f;
		out[11] = 0.0f;
		memcpy(out_pose + (size_t)bone * 12, out, sizeof(out));
	}
}
