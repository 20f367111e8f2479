// tests/cpp/shim_feature_search.cpp -- acl_b200::batch_decompressor::pack_pose_features and search_pose_features against the C calls they
// wrap: 300 requests of fabricated feature rows (S = 4, K = 4) packed with every term kind and normalisation, then searched as a database by
// 37 of its own vectors with tags and exclusion windows; the vectors and the results must be byte-identical, and each query must find a row.
// usage: shim_feature_search; prints PASS, exits 3 without a CUDA device.
#include "../../include/acl_b200/decompress.h"

#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

int main()
{
	try
	{
		acl_b200::device_context device(0);
		acl_b200::batch_decompressor batch(device);
		const uint32_t num_requests = 300, num_offsets = 4, bones_per_list = 4, num_rows = num_offsets * bones_per_list;
		std::vector<float> rows(size_t(num_requests) * num_rows * 12);
		for (size_t i = 0; i < rows.size(); ++i)
			rows[i] = std::sin(float(i) * 0.37f) * 2.0f;
		const aclb200_feature_term terms[4] = {
			{ ACLB200_FEATURE_POSITION, 1, 0, 2, 0, 7, 0.0f },
			{ ACLB200_FEATURE_VELOCITY, 0, 1, 3, 0, 5, 30.0f },
			{ ACLB200_FEATURE_DIRECTION, 2, 0, 0, 2, 5, 0.0f },
			{ ACLB200_FEATURE_POSITION, 3, 0, 0, 0, 5, 0.0f },
		};
		const uint32_t num_dims = 9, out_stride = 12, num_queries = 37;
		std::vector<float> mean(num_dims), scale(num_dims);
		for (uint32_t d = 0; d < num_dims; ++d)
		{
			mean[d] = 0.1f * float(d);
			scale[d] = 1.0f / (1.0f + float(d));
		}
		std::vector<aclb200_search_query> queries(num_queries);
		std::vector<uint32_t> tags(num_requests);
		for (uint32_t r = 0; r < num_requests; ++r)
			tags[r] = 1u << (r % 3);
		for (uint32_t q = 0; q < num_queries; ++q)
			queries[q] = aclb200_search_query{ q % 4 == 0 ? 0x7u : 0x3u, q * 8, q * 8 + (q % 5) * 3 };
		const size_t rows_bytes = rows.size() * sizeof(float), out_bytes = size_t(num_requests) * out_stride * sizeof(float);
		float* d_rows = nullptr;
		float* d_out[2] = { nullptr, nullptr };
		uint32_t* d_tags = nullptr;
		aclb200_search_query* d_queries = nullptr;
		aclb200_search_result* d_results[2] = { nullptr, nullptr };
		if (cudaMalloc(&d_rows, rows_bytes) != cudaSuccess || cudaMalloc(&d_out[0], out_bytes) != cudaSuccess
			|| cudaMalloc(&d_out[1], out_bytes) != cudaSuccess || cudaMalloc(&d_tags, num_requests * sizeof(uint32_t)) != cudaSuccess
			|| cudaMalloc(&d_queries, num_queries * sizeof(aclb200_search_query)) != cudaSuccess
			|| cudaMalloc(&d_results[0], num_queries * sizeof(aclb200_search_result)) != cudaSuccess
			|| cudaMalloc(&d_results[1], num_queries * sizeof(aclb200_search_result)) != cudaSuccess)
			return 1;
		cudaMemcpy(d_rows, rows.data(), rows_bytes, cudaMemcpyHostToDevice);
		cudaMemcpy(d_tags, tags.data(), num_requests * sizeof(uint32_t), cudaMemcpyHostToDevice);
		cudaMemcpy(d_queries, queries.data(), num_queries * sizeof(aclb200_search_query), cudaMemcpyHostToDevice);
		// the same sentinel in both buffers: the padding floats neither call writes must match too
		cudaMemset(d_out[0], 0xAB, out_bytes);
		cudaMemset(d_out[1], 0xAB, out_bytes);
		batch.pack_pose_features(d_rows, num_requests, num_offsets, bones_per_list, terms, 4, num_dims, d_out[0], out_stride, mean.data(), scale.data());
		if (aclb200_pack_pose_features(device.get(), d_rows, num_requests, num_offsets, bones_per_list, 0, terms, 4, mean.data(), scale.data(), num_dims,
			d_out[1], out_stride, nullptr) != ACLB200_OK)
			return 1;
		// queries are database vectors 5, 13, 21, ...
		batch.search_pose_features(d_out[0], num_requests, out_stride, d_out[0] + 5 * out_stride, d_queries, num_queries, 8 * out_stride, num_dims,
			d_results[0], d_tags);
		if (aclb200_search_pose_features(device.get(), d_out[1], num_requests, out_stride, d_tags, d_out[1] + 5 * out_stride, d_queries, num_queries,
			8 * out_stride, num_dims, d_results[1], nullptr) != ACLB200_OK)
			return 1;
		std::vector<uint8_t> vectors[2] = { std::vector<uint8_t>(out_bytes), std::vector<uint8_t>(out_bytes) };
		std::vector<aclb200_search_result> results[2] = { std::vector<aclb200_search_result>(num_queries), std::vector<aclb200_search_result>(num_queries) };
		for (int i = 0; i < 2; ++i)
			if (cudaMemcpy(vectors[i].data(), d_out[i], out_bytes, cudaMemcpyDeviceToHost) != cudaSuccess
				|| cudaMemcpy(results[i].data(), d_results[i], num_queries * sizeof(aclb200_search_result), cudaMemcpyDeviceToHost) != cudaSuccess)
				return 1;
		if (std::memcmp(vectors[0].data(), vectors[1].data(), out_bytes) != 0
			|| std::memcmp(results[0].data(), results[1].data(), num_queries * sizeof(aclb200_search_result)) != 0)
		{
			std::printf("FAIL shim and C call differ\n");
			return 1;
		}
		for (uint32_t q = 0; q < num_queries; ++q)
			if (results[0][q].row == ACLB200_NO_ROW || !std::isfinite(results[0][q].cost))
			{
				std::printf("FAIL query %u found no row\n", q);
				return 1;
			}
		cudaFree(d_rows);
		cudaFree(d_out[0]);
		cudaFree(d_out[1]);
		cudaFree(d_tags);
		cudaFree(d_queries);
		cudaFree(d_results[0]);
		cudaFree(d_results[1]);
	}
	catch (const acl_b200::error& e)
	{
		std::fprintf(stderr, "%s\n", e.what());
		return e.status == ACLB200_ERR_NO_DEVICE ? 3 : 1;
	}
	std::printf("PASS\n");
	return 0;
}
