/* oracle/feature_search_oracle.c -- TEST INFRASTRUCTURE ONLY: the pack and the search of motion matching (aclb200_pack_pose_features,
 * aclb200_search_pose_features) restated on the CPU, built into liboracle_feature_search.so by oracle/feature_search.mk. The direction term
 * needs rtm_quat_mul_vector3, which is file-local to acl_oracle.c, so that file is compiled in here unchanged. */
#include "acl_oracle.c"

#include <math.h>

typedef struct aclo_feature_term
{
	uint32_t kind, s0, s1, k, axis, components;
	float inv_dt;
} aclo_feature_term;

typedef struct aclo_search_query
{
	uint32_t tag_mask, exclude_begin, exclude_end;
} aclo_search_query;

typedef struct aclo_search_result
{
	uint32_t row;
	float cost;
} aclo_search_result;

/* rtm::quat_mul_vector3(e_axis, rotation), the unit vector as it is */
void aclo_feature_direction(const float* rotation, uint32_t axis, float* out)
{
	const float e[3] = { axis == 0 ? 1.0f : 0.0f, axis == 1 ? 1.0f : 0.0f, axis == 2 ? 1.0f : 0.0f };
	rtm_quat_mul_vector3(e, rotation, out);
}

/* out[r][d] = (v_d - mean[d]) * scale[d] for the rows of request r at rows + r * pose_stride (bytes), row (s, k) at (s * K + k) * 48. The
 * terms are taken as valid (the library refuses the others). Returns the number of dimensions written. */
uint32_t aclo_pack_pose_features(const uint8_t* rows, uint32_t num_requests, uint32_t bones_per_list, uint64_t pose_stride,
	const aclo_feature_term* terms, uint32_t num_terms, const float* mean, const float* scale, float* out, uint64_t out_stride)
{
	uint32_t num_dims = 0;
	for (uint32_t r = 0; r < num_requests; ++r)
	{
		const uint8_t* pose = rows + r * pose_stride;
		uint32_t d = 0;
		for (uint32_t t = 0; t < num_terms; ++t)
		{
			const aclo_feature_term* term = &terms[t];
			const float* first = (const float*)(pose + (size_t)(term->s0 * bones_per_list + term->k) * 48);
			const float* second = (const float*)(pose + (size_t)(term->s1 * bones_per_list + term->k) * 48);
			float direction[3] = { 0.0f, 0.0f, 0.0f };
			if (term->kind == 1)
				aclo_feature_direction(first, term->axis, direction);
			for (uint32_t c = 0; c < 3; ++c)
			{
				if ((term->components & (1u << c)) == 0)
					continue;
				float v;
				if (term->kind == 0)
					v = first[4 + c];
				else if (term->kind == 1)
					v = direction[c];
				else
				{
					const float delta = second[4 + c] - first[4 + c];
					v = delta * term->inv_dt;
				}
				const float centred = v - (mean != NULL ? mean[d] : 0.0f);
				out[r * out_stride + d] = centred * (scale != NULL ? scale[d] : 1.0f);
				++d;
			}
		}
		num_dims = d;
	}
	return num_dims;
}

/* acc = +0; acc = fmaf(q[d] - x[d], q[d] - x[d], acc) for d in order */
float aclo_feature_cost(const float* query, const float* row, uint32_t num_dims)
{
	float acc = 0.0f;
	for (uint32_t d = 0; d < num_dims; ++d)
	{
		const float diff = query[d] - row[d];
		acc = fmaf(diff, diff, acc);
	}
	return acc;
}

/* The candidate with the smallest cost, the lowest row on a tie; {0xFFFFFFFF, +inf} without one */
void aclo_search_pose_features(const float* database, uint64_t num_rows, uint64_t db_stride, const uint32_t* row_tags, const float* query_vectors,
	const aclo_search_query* queries, uint32_t num_queries, uint64_t q_stride, uint32_t num_dims, aclo_search_result* results)
{
	for (uint32_t q = 0; q < num_queries; ++q)
	{
		aclo_search_result best = { 0xFFFFFFFFu, INFINITY };
		for (uint64_t r = 0; r < num_rows; ++r)
		{
			const uint32_t tag = row_tags != NULL ? row_tags[r] : 0xFFFFFFFFu;
			if ((tag & queries[q].tag_mask) == 0 || (r >= queries[q].exclude_begin && r < queries[q].exclude_end))
				continue;
			const float cost = aclo_feature_cost(query_vectors + q * q_stride, database + r * db_stride, num_dims);
			if (isnan(cost))
				continue;
			if (cost < best.cost || best.row == 0xFFFFFFFFu)
			{
				best.row = (uint32_t)r;
				best.cost = cost;
			}
		}
		results[q] = best;
	}
}
