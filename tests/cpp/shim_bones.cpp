// tests/cpp/shim_bones.cpp -- acl_b200::batch_decompressor::decompress_bones against the C call it wraps: 64 requests of the clip over
// two bone lists picked per request (a leaf list and one with a duplicate and an ACLB200_NO_BONE hole), local QVV48 rows, qvvf and matrix
// rows on a binary tree; the outputs must be byte-identical.
// usage: shim_bones <clip.acl.bin>; prints PASS, exits 3 without a CUDA device.
#include "../../include/acl_b200/decompress.h"

#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <fstream>
#include <iterator>
#include <vector>

int main(int argc, char** argv)
{
	if (argc != 2)
		return 2;
	std::ifstream file(argv[1], std::ios::binary);
	const std::vector<char> blob((std::istreambuf_iterator<char>(file)), std::istreambuf_iterator<char>());
	try
	{
		acl_b200::device_context device(0);
		acl_b200::batch_decompressor batch(device);
		const void* pointer = blob.data();
		const uint32_t size = uint32_t(blob.size());
		if (!batch.upload(&pointer, &size, 1))
			return 1;
		const uint32_t num_tracks = batch.info().max_tracks;
		const uint32_t bones_per_list = 4;
		const uint32_t num_requests = 64;
		std::vector<aclb200_request> requests;
		std::vector<uint32_t> request_lists;
		for (uint32_t i = 0; i < num_requests; ++i)
		{
			requests.push_back(aclb200_request{ 0u, float(i) * 0.037f - 0.1f });
			request_lists.push_back(i % 3);		// list 2 does not exist: those requests write nothing
		}
		const std::vector<uint32_t> bone_lists = { num_tracks - 1, num_tracks / 2, num_tracks / 3, 0u,
			num_tracks - 1, ACLB200_NO_BONE, num_tracks - 1, num_tracks };
		std::vector<uint32_t> parents(num_tracks);
		for (uint32_t bone = 0; bone < num_tracks; ++bone)
			parents[bone] = bone == 0 ? 0xFFFFFFFFu : (bone - 1) / 2;
		const size_t out_bytes = size_t(num_requests) * bones_per_list * 48;
		aclb200_request* d_requests = nullptr;
		uint32_t* d_request_lists = nullptr;
		uint32_t* d_bone_lists = nullptr;
		uint32_t* d_parents = nullptr;
		uint8_t* d_out[2] = { nullptr, nullptr };
		if (cudaMalloc(&d_requests, requests.size() * sizeof(aclb200_request)) != cudaSuccess
			|| cudaMalloc(&d_request_lists, request_lists.size() * sizeof(uint32_t)) != cudaSuccess
			|| cudaMalloc(&d_bone_lists, bone_lists.size() * sizeof(uint32_t)) != cudaSuccess
			|| cudaMalloc(&d_parents, num_tracks * sizeof(uint32_t)) != cudaSuccess || cudaMalloc(&d_out[0], out_bytes) != cudaSuccess
			|| cudaMalloc(&d_out[1], out_bytes) != cudaSuccess)
			return 1;
		cudaMemcpy(d_requests, requests.data(), requests.size() * sizeof(aclb200_request), cudaMemcpyHostToDevice);
		cudaMemcpy(d_request_lists, request_lists.data(), request_lists.size() * sizeof(uint32_t), cudaMemcpyHostToDevice);
		cudaMemcpy(d_bone_lists, bone_lists.data(), bone_lists.size() * sizeof(uint32_t), cudaMemcpyHostToDevice);
		cudaMemcpy(d_parents, parents.data(), num_tracks * sizeof(uint32_t), cudaMemcpyHostToDevice);
		aclb200_options options;
		aclb200_default_options(&options);
		const auto same = [&](const char* what) -> bool
		{
			std::vector<uint8_t> got[2] = { std::vector<uint8_t>(out_bytes), std::vector<uint8_t>(out_bytes) };
			for (int i = 0; i < 2; ++i)
				if (cudaMemcpy(got[i].data(), d_out[i], out_bytes, cudaMemcpyDeviceToHost) != cudaSuccess)
					return false;
			if (std::memcmp(got[0].data(), got[1].data(), out_bytes) == 0)
				return true;
			std::printf("FAIL %s\n", what);
			return false;
		};
		struct Case { const char* what; const uint32_t* parents; uint32_t kind; };
		const Case cases[] = { { "local", nullptr, ACLB200_OBJECT_QVVF }, { "qvvf", d_parents, ACLB200_OBJECT_QVVF },
			{ "matrix", d_parents, ACLB200_OBJECT_MATRIX3X4F } };
		for (const Case& c : cases)
		{
			// the same sentinel in both buffers: the rows neither call writes must match too
			cudaMemset(d_out[0], 0xAB, out_bytes);
			cudaMemset(d_out[1], 0xAB, out_bytes);
			batch.decompress_bones(d_requests, num_requests, options, d_bone_lists, 2, bones_per_list, d_out[0], d_request_lists, c.parents, nullptr,
				c.kind);
			if (aclb200_decompress_bones(device.get(), batch.clipset(), d_requests, num_requests, &options, d_bone_lists, 2, bones_per_list,
				d_request_lists, c.parents, nullptr, c.kind, d_out[1], nullptr, nullptr) != ACLB200_OK)
				return 1;
			if (!same(c.what))
				return 1;
		}
		cudaFree(d_requests);
		cudaFree(d_request_lists);
		cudaFree(d_bone_lists);
		cudaFree(d_parents);
		cudaFree(d_out[0]);
		cudaFree(d_out[1]);
	}
	catch (const acl_b200::error& e)
	{
		std::fprintf(stderr, "%s\n", e.what());
		return e.status == ACLB200_ERR_NO_DEVICE ? 3 : 1;
	}
	std::printf("PASS\n");
	return 0;
}
