/* oracle/mirror_oracle.c -- TEST INFRASTRUCTURE ONLY: mirroring (aclb200_mirror_poses, and the mirror step of
 * aclb200_decompress_tracks_mirrored) restated on the CPU, built into liboracle_mirror.so by oracle/mirror.mk. rtm_quat_mul and
 * rtm_quat_mul_vector3 are file-local to acl_oracle.c, so that file is compiled in here unchanged. */
#include "acl_oracle.c"

/* aclb200_mirror_entry: pre, post (xyzw), the mirror row, three ignored words; 48 bytes */
typedef struct aclo_mirror_entry
{
	float pre[4];
	float post[4];
	uint32_t mirror;
	uint32_t reserved[3];
} aclo_mirror_entry;

static float flip_sign(float v, int flip) { return u32_as_f32(f32_as_u32(v) ^ (flip ? 0x80000000u : 0u)); }

/* row i's partner among n rows: m = table[i].mirror when m < n and table[m].mirror == i, else i itself (*invalid set) */
uint32_t aclo_mirror_partner(const aclo_mirror_entry* table, uint32_t i, uint32_t n, int* invalid)
{
	const uint32_t m = table[i].mirror;
	if (m < n && table[m].mirror == i)
		return m;
	*invalid = 1;
	return i;
}

/* the mirrored row from the partner's QVV48 row `src` and this row's entry: rotation quat_mul(quat_mul(pre, reflect_q(q)), post),
 * translation quat_mul_vector3(reflect_t(t), post), scale copied, w lanes 0 */
void aclo_mirror_row(const float* src, const aclo_mirror_entry* entry, uint32_t axis, float* out)
{
	const float reflected[4] = { flip_sign(src[0], axis != 0), flip_sign(src[1], axis != 1), flip_sign(src[2], axis != 2), src[3] };
	const float t[3] = { flip_sign(src[4], axis == 0), flip_sign(src[5], axis == 1), flip_sign(src[6], axis == 2) };
	float inner[4], row[12];
	rtm_quat_mul(entry->pre, reflected, inner);
	rtm_quat_mul(inner, entry->post, row);
	rtm_quat_mul_vector3(t, entry->post, row + 4);
	row[7] = 0.0f;
	memcpy(row + 8, src + 8, 3 * sizeof(float));
	row[11] = 0.0f;
	memcpy(out, row, sizeof(row));
}

/* one pose of n QVV48 rows mirrored with the table: out may be pose. Returns ACLB200_ERROR_FLAG_INVALID_MIRROR (8) when a row had no
 * partner, else 0. */
uint32_t aclo_mirror_pose(const float* pose, const aclo_mirror_entry* table, uint32_t n, uint32_t axis, float* out)
{
	float* rows = (float*)malloc((size_t)n * 12 * sizeof(float) + 1);
	uint32_t flags = 0;
	for (uint32_t i = 0; i < n; ++i)
	{
		int invalid = 0;
		const uint32_t m = aclo_mirror_partner(table, i, n, &invalid);
		if (invalid)
			flags = 8u;
		aclo_mirror_row(pose + (size_t)m * 12, table + i, axis, rows + (size_t)i * 12);
	}
	memcpy(out, rows, (size_t)n * 12 * sizeof(float));
	free(rows);
	return flags;
}
