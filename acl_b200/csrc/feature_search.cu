// acl_b200/csrc/feature_search.cu -- motion matching on pose features: the pack (aclb200_pack_pose_features) turns the 48 byte rows of
// aclb200_extract_pose_features into weighted float vectors, the search (aclb200_search_pose_features) finds each query's lowest cost
// allowed database row.
//
// Pack: one thread per output float (request r, dimension d). The host resolves the terms into one PackDim per dimension (kind, rows,
// component, inv_dt, mean, scale), so a thread reads one or two row fields, or one rotation for a direction, and stores one float.
//
// Search: a result is the minimum of the 64 bit key (cost bits << 32) | row over a query's candidates. Costs are never negative (an FMA
// chain of squares from +0), so their bits order like their values, and a tie goes to the lower row; the aclb200_search_result {row, cost}
// read as a little endian uint64 IS that key. A NaN cost's key lies above every other, {NO_ROW, +inf}'s included, so it never wins. One
// kernel writes every result as {ACLB200_NO_ROW, +inf} (the key 0x7F800000FFFFFFFF), then every block of the search atomicMin-s its per
// query best into the results. The minimum does not depend on which block saw which rows, nor on their order: any tiling gives the same
// bits.
//
// Search tiling: a block holds a tile of BQ = QG * TQ queries in shared memory (dimension major) for its whole life and walks a range of
// BR = RG * TR row tiles, each staged in shared memory dimension major too. Thread (qg, rg) keeps TQ x TR costs in registers: per
// dimension it reads TQ query values and TR row values and runs TQ * TR subtract + FMA pairs. The grid is (query tiles) x (row splits),
// with just enough row splits to fill the device once; each block keeps its TQ running minima in registers and reduces them through
// shared memory into one atomicMin per query at its end.
#include "object_space.cuh"

#include <algorithm>

namespace aclb200
{
	namespace
	{
		__global__ void __launch_bounds__(256) pack_pose_features_kernel(const PackParams p)
		{
			const uint64_t index = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
			if (index >= uint64_t(p.num_requests) * p.num_dims)
				return;
			const uint32_t request = uint32_t(index / p.num_dims);
			const uint32_t d = uint32_t(index - uint64_t(request) * p.num_dims);
			const PackDim& dim = p.dims[d];
			const uint8_t* pose = p.rows + uint64_t(request) * p.pose_stride;
			const float* first = reinterpret_cast<const float*>(pose + dim.row0 * 48u);
			float value;
			if (dim.kind == ACLB200_FEATURE_POSITION)
				value = __ldg(first + 4 + dim.component);
			else if (dim.kind == ACLB200_FEATURE_VELOCITY)
			{
				const float* second = reinterpret_cast<const float*>(pose + dim.row1 * 48u);
				value = __fmul_rn(__fsub_rn(__ldg(second + 4 + dim.component), __ldg(first + 4 + dim.component)), dim.inv_dt);
			}
			else
			{
				// rtm::quat_mul_vector3(e_axis, rotation): the object space function, on the unit vector as it is
				const float4 q = __ldg(reinterpret_cast<const float4*>(first));
				const obj::Vec3<float> axis = { dim.axis == 0 ? 1.0f : 0.0f, dim.axis == 1 ? 1.0f : 0.0f, dim.axis == 2 ? 1.0f : 0.0f };
				const obj::Vec3<float> v = obj::quat_mul_vector3(obj::Fp<float>{}, axis, obj::Quat<float>{ q.x, q.y, q.z, q.w });
				value = dim.component == 0 ? v.x : dim.component == 1 ? v.y : v.z;
			}
			p.out[uint64_t(request) * p.out_stride + d] = __fmul_rn(__fsub_rn(value, dim.mean), dim.scale);
		}

		constexpr unsigned long long k_no_result = 0x7F800000FFFFFFFFull;		// {ACLB200_NO_ROW, +inf}
		constexpr uint32_t k_search_threads = 256;

		__global__ void __launch_bounds__(256) clear_search_results_kernel(unsigned long long* results, uint32_t num_queries)
		{
			const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
			if (q < num_queries)
				results[q] = k_no_result;
		}

		// stages `count` vectors of D floats (rows first .. first + count - 1 of `base`, `stride` floats apart) into s[d * width + i]; vectors at
		// or beyond `limit` are zeros
		template<uint32_t WIDTH>
		__device__ __forceinline__ void stage_vectors(float* s, const float* base, uint64_t stride, uint64_t first, uint64_t limit, uint32_t num_dims)
		{
			const uint32_t chunks = (num_dims + 3) / 4;
			for (uint32_t item = threadIdx.x; item < WIDTH * chunks; item += k_search_threads)
			{
				const uint32_t i = item % WIDTH;
				const uint32_t c = item / WIDTH;
				const uint64_t vector = first + i;
				float4 v = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
				if (vector < limit)
					v = __ldg(reinterpret_cast<const float4*>(base + vector * stride) + c);
				const float lanes[4] = { v.x, v.y, v.z, v.w };
				#pragma unroll
				for (uint32_t k = 0; k < 4; ++k)
					if (c * 4 + k < num_dims)
						s[(c * 4 + k) * WIDTH + i] = lanes[k];
			}
		}

		// the 8 byte slots of a block's per query keys: an even number
		__host__ __device__ constexpr uint32_t k_best_slots(uint32_t queries_per_block)
		{
			return (queries_per_block + 1) & ~1u;
		}

		template<uint32_t TQ, uint32_t TR, uint32_t QG, uint32_t RG>
		__global__ void __launch_bounds__(k_search_threads) search_pose_features_kernel(const SearchParams p)
		{
			static_assert(QG * RG == k_search_threads, "one thread per (query group, row group)");
			constexpr uint32_t BQ = QG * TQ, BR = RG * TR;
			extern __shared__ __align__(16) unsigned long long s_search[];
			unsigned long long* s_best = s_search;						// [BQ], first: 8 byte keys, and 16 bytes of them keep the
			float* s_query = reinterpret_cast<float*>(s_best + k_best_slots(BQ));	// floats after them 16 byte aligned; [D][BQ]
			float* s_row = s_query + p.num_dims * BQ;					// [D][BR]
			uint32_t* s_tag = reinterpret_cast<uint32_t*>(s_row + p.num_dims * BR);		// [BR]
			uint32_t* s_info = s_tag + BR;								// [BQ][3] tag mask, exclude_begin, exclude_end

			const uint32_t first_query = blockIdx.x * BQ;
			stage_vectors<BQ>(s_query, p.query_vectors, p.q_stride, first_query, p.num_queries, p.num_dims);
			for (uint32_t i = threadIdx.x; i < BQ; i += k_search_threads)
			{
				const uint32_t query = first_query + i;
				// a query past the end allows no tag: it never has a candidate
				const aclb200_search_query info = query < p.num_queries ? p.queries[query] : aclb200_search_query{ 0u, 0u, 0u };
				s_info[i * 3] = info.tag_mask;
				s_info[i * 3 + 1] = info.exclude_begin;
				s_info[i * 3 + 2] = info.exclude_end;
				s_best[i] = k_no_result;
			}

			const uint32_t qg = threadIdx.x / RG, rg = threadIdx.x % RG;
			const uint64_t num_tiles = (p.num_rows + BR - 1) / BR;
			const uint64_t tile_begin = num_tiles * blockIdx.y / gridDim.y;
			const uint64_t tile_end = num_tiles * (blockIdx.y + 1) / gridDim.y;
			unsigned long long best[TQ];
			#pragma unroll
			for (uint32_t i = 0; i < TQ; ++i)
				best[i] = k_no_result;

			for (uint64_t tile = tile_begin; tile < tile_end; ++tile)
			{
				const uint64_t first_row = tile * BR;
				__syncthreads();		// the previous tile's rows are read
				stage_vectors<BR>(s_row, p.database, p.db_stride, first_row, p.num_rows, p.num_dims);
				for (uint32_t i = threadIdx.x; i < BR; i += k_search_threads)
					// a row past the end has no tag: no query allows it
					s_tag[i] = first_row + i >= p.num_rows ? 0u : p.row_tags != nullptr ? __ldg(p.row_tags + first_row + i) : 0xFFFFFFFFu;
				__syncthreads();

				float cost[TQ][TR];
				#pragma unroll
				for (uint32_t i = 0; i < TQ; ++i)
					#pragma unroll
					for (uint32_t j = 0; j < TR; ++j)
						cost[i][j] = 0.0f;
				for (uint32_t d = 0; d < p.num_dims; ++d)
				{
					float q[TQ], x[TR];
					#pragma unroll
					for (uint32_t i = 0; i < TQ; ++i)
						q[i] = s_query[d * BQ + qg * TQ + i];
					#pragma unroll
					for (uint32_t j = 0; j < TR; ++j)
						x[j] = s_row[d * BR + rg * TR + j];
					#pragma unroll
					for (uint32_t i = 0; i < TQ; ++i)
						#pragma unroll
						for (uint32_t j = 0; j < TR; ++j)
						{
							const float diff = __fsub_rn(q[i], x[j]);
							cost[i][j] = __fmaf_rn(diff, diff, cost[i][j]);
						}
				}

				#pragma unroll
				for (uint32_t j = 0; j < TR; ++j)
				{
					const uint32_t local_row = rg * TR + j;
					const uint32_t row = uint32_t(first_row) + local_row;		// N < 2^32 - 1
					const uint32_t tag = s_tag[local_row];
					#pragma unroll
					for (uint32_t i = 0; i < TQ; ++i)
					{
						const uint32_t* info = s_info + (qg * TQ + i) * 3;
						const bool excluded = row >= info[1] && row < info[2];
						if ((tag & info[0]) != 0 && !excluded)
						{
							// a NaN cost needs no test: every NaN's bits (either sign) lie above +inf's, so its key is above
							// k_no_result and never wins
							const unsigned long long key = (static_cast<unsigned long long>(__float_as_uint(cost[i][j])) << 32) | row;
							best[i] = key < best[i] ? key : best[i];
						}
					}
				}
			}

			#pragma unroll
			for (uint32_t i = 0; i < TQ; ++i)
				if (best[i] != k_no_result)
					atomicMin(s_best + qg * TQ + i, best[i]);
			__syncthreads();
			for (uint32_t i = threadIdx.x; i < BQ; i += k_search_threads)
				if (s_best[i] != k_no_result)
					atomicMin(reinterpret_cast<unsigned long long*>(p.results + first_query + i), s_best[i]);
		}

		// The three shapes: one query (the database split over the whole device), a few queries, and many queries (a 128 x 64 tile per block)
		struct SearchShape
		{
			void (*kernel)(SearchParams);
			uint32_t queries_per_block;
			uint32_t rows_per_block;
		};
		const SearchShape k_search_shapes[3] = {
			{ search_pose_features_kernel<1, 1, 1, 256>, 1, 256 },
			{ search_pose_features_kernel<4, 4, 4, 64>, 16, 256 },
			{ search_pose_features_kernel<8, 4, 16, 16>, 128, 64 },
		};

		const SearchShape& search_shape(uint32_t num_queries)
		{
			return k_search_shapes[num_queries == 1 ? 0 : num_queries <= 64 ? 1 : 2];
		}

		uint32_t search_smem_bytes(const SearchShape& shape, uint32_t num_dims)
		{
			return k_best_slots(shape.queries_per_block) * 8
				+ (num_dims * (shape.queries_per_block + shape.rows_per_block) + shape.rows_per_block + 3 * shape.queries_per_block) * 4;
		}
	}

	cudaError_t configure_feature_search_kernels()
	{
		cudaError_t error = cudaSuccess;
		for (const SearchShape& shape : k_search_shapes)
			if (error == cudaSuccess)
				error = cudaFuncSetAttribute(shape.kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(search_smem_bytes(shape, ACLB200_MAX_FEATURE_DIMS)));
		return error;
	}

	cudaError_t launch_pack_pose_features(const PackParams& params, cudaStream_t stream)
	{
		const uint64_t items = uint64_t(params.num_requests) * params.num_dims;
		pack_pose_features_kernel<<<uint32_t((items + 255) / 256), 256, 0, stream>>>(params);
		return cudaGetLastError();
	}

	cudaError_t launch_search_pose_features(const SearchParams& params, int num_sms, cudaStream_t stream)
	{
		clear_search_results_kernel<<<(params.num_queries + 255) / 256, 256, 0, stream>>>(reinterpret_cast<unsigned long long*>(params.results),
			params.num_queries);
		cudaError_t error = cudaGetLastError();
		if (error != cudaSuccess || params.num_rows == 0)
			return error;
		const SearchShape& shape = search_shape(params.num_queries);
		const uint32_t smem = search_smem_bytes(shape, params.num_dims);
		int resident = 0;
		error = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, shape.kernel, k_search_threads, smem);
		if (error != cudaSuccess)
			return error;
		// enough row splits that the grid fills every SM once, never more splits than row tiles
		const uint32_t query_tiles = (params.num_queries + shape.queries_per_block - 1) / shape.queries_per_block;
		const uint64_t row_tiles = (params.num_rows + shape.rows_per_block - 1) / shape.rows_per_block;
		const uint64_t slots = uint64_t(num_sms) * uint32_t(resident > 0 ? resident : 1);
		const uint64_t splits = std::max<uint64_t>(1, std::min<uint64_t>(row_tiles, slots / query_tiles));
		shape.kernel<<<dim3(query_tiles, uint32_t(splits)), k_search_threads, smem, stream>>>(params);
		return cudaGetLastError();
	}
}
