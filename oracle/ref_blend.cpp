// oracle/ref_blend.cpp -- TEST INFRASTRUCTURE ONLY: rtm::qvv_lerp from the unmodified reference's math library, compiled into
// _ref/libaclref_blend.so (oracle/blend.mk) with the flags of the reference build (-msse4.1: quat_lerp's dpps path) where the reference
// tree exists.
#include <rtm/qvvf.h>

#include <cstddef>
#include <cstdint>

extern "C"
{
	// rtm::qvv_lerp(from, to, weight) (qvvf.h:439-445) on every bone of one pose: [num_tracks][12] rtm::qvvf rows in (rotation xyzw,
	// translation xyz + w, scale xyz + w), out [num_tracks][12] as rtm leaves them
	__attribute__((visibility("default"))) void aclref_qvv_lerp(const float* from_pose, const float* to_pose, uint32_t num_tracks, float weight,
		float* out)
	{
		for (uint32_t bone = 0; bone < num_tracks; ++bone)
		{
			const float* f = from_pose + size_t(bone) * 12;
			const float* t = to_pose + size_t(bone) * 12;
			const rtm::qvvf from = rtm::qvv_set(rtm::quat_load(f), rtm::vector_load(f + 4), rtm::vector_load(f + 8));
			const rtm::qvvf to = rtm::qvv_set(rtm::quat_load(t), rtm::vector_load(t + 4), rtm::vector_load(t + 8));
			const rtm::qvvf result = rtm::qvv_lerp(from, to, weight);
			float* o = out + size_t(bone) * 12;
			rtm::quat_store(result.rotation, o);
			rtm::vector_store(result.translation, o + 4);
			rtm::vector_store(result.scale, o + 8);
		}
	}
}
