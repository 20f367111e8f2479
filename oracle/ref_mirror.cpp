// oracle/ref_mirror.cpp -- TEST INFRASTRUCTURE ONLY: the mirrored row built from the unmodified reference's rtm::quat_mul and
// rtm::quat_mul_vector3, compiled into _ref/libaclref_mirror.so (oracle/mirror.mk) with the flags of the reference build where the
// reference tree exists. The reflections are sign bit flips and the partner rule plain integer tests, as the project specifies them.
#include <rtm/quatf.h>
#include <rtm/vector4f.h>

#include <cstddef>
#include <cstdint>
#include <cstdlib>
#include <cstring>

namespace
{
	struct mirror_entry
	{
		float pre[4];
		float post[4];
		uint32_t mirror;
		uint32_t reserved[3];
	};

	float flip_sign(float v, bool flip)
	{
		uint32_t bits;
		std::memcpy(&bits, &v, 4);
		bits ^= flip ? 0x80000000u : 0u;
		std::memcpy(&v, &bits, 4);
		return v;
	}

	void mirror_row(const float* src, const mirror_entry& entry, uint32_t axis, float* out)
	{
		const rtm::quatf reflected = rtm::quat_set(flip_sign(src[0], axis != 0), flip_sign(src[1], axis != 1), flip_sign(src[2], axis != 2), src[3]);
		const rtm::vector4f t = rtm::vector_set(flip_sign(src[4], axis == 0), flip_sign(src[5], axis == 1), flip_sign(src[6], axis == 2), 0.0f);
		const rtm::quatf pre = rtm::quat_load(entry.pre);
		const rtm::quatf post = rtm::quat_load(entry.post);
		float row[12];
		rtm::quat_store(rtm::quat_mul(rtm::quat_mul(pre, reflected), post), row);
		rtm::vector_store3(rtm::quat_mul_vector3(t, post), row + 4);
		row[7] = 0.0f;
		std::memcpy(row + 8, src + 8, 3 * sizeof(float));
		row[11] = 0.0f;
		std::memcpy(out, row, sizeof(row));
	}
}

extern "C"
{
	// one pose of n QVV48 rows mirrored with the table (48 byte entries); returns 8 when a row had no partner
	__attribute__((visibility("default"))) uint32_t aclref_mirror_pose(const float* pose, const void* table_bytes, uint32_t n, uint32_t axis,
		float* out)
	{
		const mirror_entry* table = static_cast<const mirror_entry*>(table_bytes);
		float* rows = static_cast<float*>(std::malloc(size_t(n) * 12 * sizeof(float) + 1));
		uint32_t flags = 0;
		for (uint32_t i = 0; i < n; ++i)
		{
			uint32_t m = table[i].mirror;
			if (!(m < n && table[m].mirror == i))
			{
				m = i;
				flags = 8u;
			}
			mirror_row(pose + size_t(m) * 12, table[i], axis, rows + size_t(i) * 12);
		}
		std::memcpy(out, rows, size_t(n) * 12 * sizeof(float));
		std::free(rows);
		return flags;
	}
}
