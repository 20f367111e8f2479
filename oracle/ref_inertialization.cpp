// oracle/ref_inertialization.cpp -- TEST INFRASTRUCTURE ONLY: the inertialization capture and apply built from the unmodified reference's
// rtm::quat_rotation_log, quat_rotation_exp, quat_mul and quat_conjugate, compiled into _ref/libaclref_inertialization.so
// (oracle/inertialization.mk) with the flags of the reference build where the reference tree exists. abs() and the spring are plain float
// arithmetic (-ffp-contract=off), as the project specifies them.
#include <rtm/quatf.h>
#include <rtm/vector4f.h>

#include <cstddef>
#include <cstdint>

namespace
{
	rtm::quatf load_rotation(const float* row) { return rtm::quat_load(row); }

	// 2 log(abs(quat_mul(conj(from), to))).xyz
	void scaled_angle_axis_between(const float* from, const float* to, float out[3])
	{
		rtm::quatf q = rtm::quat_mul(rtm::quat_conjugate(load_rotation(from)), load_rotation(to));
		if (rtm::quat_get_w(q) < 0.0f)
			q = rtm::quat_neg(q);
		float l[4];
		rtm::quat_store(rtm::quat_rotation_log(q), l);
		for (int i = 0; i < 3; ++i)
			out[i] = 2.0f * l[i];
	}
}

extern "C"
{
	// rtm::quat_rotation_log(q) / quat_rotation_exp(q) of one xyzw quaternion, all four lanes as rtm leaves them
	__attribute__((visibility("default"))) void aclref_quat_rotation_log(const float* q, float* out)
	{
		rtm::quat_store(rtm::quat_rotation_log(rtm::quat_load(q)), out);
	}

	__attribute__((visibility("default"))) void aclref_quat_rotation_exp(const float* q, float* out)
	{
		rtm::quat_store(rtm::quat_rotation_exp(rtm::quat_load(q)), out);
	}

	// the capture of one transition: [num_tracks][12] rows in, [num_tracks][16] record entries out
	__attribute__((visibility("default"))) void aclref_begin_inertialization(const float* src, const float* src_prev, const float* dst,
		const float* dst_prev, uint32_t num_tracks, float inv_dt, float* record)
	{
		for (uint32_t bone = 0; bone < num_tracks; ++bone)
		{
			const float* s = src + size_t(bone) * 12;
			const float* sp = src_prev + size_t(bone) * 12;
			const float* d = dst + size_t(bone) * 12;
			const float* dp = dst_prev + size_t(bone) * 12;
			float* e = record + size_t(bone) * 16;
			float rot_x[3], src_w[3], dst_w[3];
			scaled_angle_axis_between(d, s, rot_x);
			scaled_angle_axis_between(sp, s, src_w);
			scaled_angle_axis_between(dp, d, dst_w);
			for (int i = 0; i < 3; ++i)
			{
				e[i] = rot_x[i];
				e[4 + i] = src_w[i] * inv_dt - dst_w[i] * inv_dt;
				e[8 + i] = s[4 + i] - d[4 + i];
				e[12 + i] = (s[4 + i] - sp[4 + i]) * inv_dt - (d[4 + i] - dp[4 + i]) * inv_dt;
			}
			e[3] = e[7] = e[11] = e[15] = 0.0f;
		}
	}

	// the apply on one pose with one record: [num_tracks][12] rows in and out
	__attribute__((visibility("default"))) void aclref_inertialize_pose(const float* pose, const float* record, uint32_t num_tracks, float elapsed,
		float halflife, float* out)
	{
		const float y = (2.7725887f / (halflife + 1e-5f)) * 0.5f;
		const float u = y * elapsed;
		const float e = 1.0f / (((1.0f + u) + (0.48f * u) * u) + ((0.235f * u) * u) * u);
		for (uint32_t bone = 0; bone < num_tracks; ++bone)
		{
			const float* d = pose + size_t(bone) * 12;
			const float* r = record + size_t(bone) * 16;
			float half_offset[4] = { 0.0f, 0.0f, 0.0f, 0.0f };
			float* o = out + size_t(bone) * 12;
			float translation[3];
			for (int i = 0; i < 3; ++i)
			{
				half_offset[i] = (e * (r[i] + (r[4 + i] + r[i] * y) * elapsed)) * 0.5f;
				translation[i] = d[4 + i] + e * (r[8 + i] + (r[12 + i] + r[8 + i] * y) * elapsed);
			}
			const rtm::quatf offset = rtm::quat_rotation_exp(rtm::quat_load(half_offset));
			rtm::quat_store(rtm::quat_mul(load_rotation(d), offset), o);
			for (int i = 0; i < 3; ++i)
			{
				o[4 + i] = translation[i];
				o[8 + i] = d[8 + i];
			}
			o[7] = 0.0f;
			o[11] = 0.0f;
		}
	}
}
