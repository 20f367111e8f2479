// tests/cpp/shim_features.cpp -- acl_b200::batch_decompressor::extract_pose_features against the C call it wraps: 48 requests of the clip
// (clamped and looping, one with an invalid looping value that writes nothing) at four offsets, a list of four bones with a hole, a binary
// tree skeleton, the root at track 0 and at the clip's last track; the outputs and the flags must be byte-identical.
// usage: shim_features <clip.acl.bin>; prints PASS, exits 3 without a CUDA device.
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
		const uint32_t num_requests = 48;
		const float offsets[4] = { -1.0f / 30.0f, 0.0f, 1.0f / 3.0f, 2.0f / 3.0f };
		const uint32_t num_offsets = 4, bones_per_list = 4;
		std::vector<aclb200_feature_request> requests;
		for (uint32_t i = 0; i < num_requests; ++i)
			requests.push_back(aclb200_feature_request{ 0u, float(i) * 0.061f - 0.2f, i % 2 });
		requests[7].looping = 2;		// writes nothing
		std::vector<uint32_t> parents(num_tracks);
		for (uint32_t b = 0; b < num_tracks; ++b)
			parents[b] = b == 0 ? 0xFFFFFFFFu : (b - 1) / 2;
		const uint32_t bones[4] = { 0, num_tracks - 1, ACLB200_NO_BONE, num_tracks / 2 };
		const size_t out_bytes = size_t(num_requests) * num_offsets * bones_per_list * 48;
		aclb200_feature_request* d_requests = nullptr;
		uint32_t* d_bones = nullptr;
		uint32_t* d_parents = nullptr;
		uint32_t* d_roots = nullptr;
		uint32_t* d_flags = nullptr;
		uint8_t* d_out[2] = { nullptr, nullptr };
		const uint32_t last = num_tracks - 1;
		if (cudaMalloc(&d_requests, requests.size() * sizeof(aclb200_feature_request)) != cudaSuccess
			|| cudaMalloc(&d_bones, sizeof(bones)) != cudaSuccess || cudaMalloc(&d_parents, num_tracks * sizeof(uint32_t)) != cudaSuccess
			|| cudaMalloc(&d_roots, sizeof(uint32_t)) != cudaSuccess || cudaMalloc(&d_flags, 2 * sizeof(uint32_t)) != cudaSuccess
			|| cudaMalloc(&d_out[0], out_bytes) != cudaSuccess || cudaMalloc(&d_out[1], out_bytes) != cudaSuccess)
			return 1;
		cudaMemcpy(d_requests, requests.data(), requests.size() * sizeof(aclb200_feature_request), cudaMemcpyHostToDevice);
		cudaMemcpy(d_bones, bones, sizeof(bones), cudaMemcpyHostToDevice);
		cudaMemcpy(d_parents, parents.data(), num_tracks * sizeof(uint32_t), cudaMemcpyHostToDevice);
		cudaMemcpy(d_roots, &last, sizeof(uint32_t), cudaMemcpyHostToDevice);
		aclb200_options options;
		aclb200_default_options(&options);
		options.looping_policy = ACLB200_LOOP_CLAMP;
		const uint32_t* roots[] = { nullptr, d_roots };
		for (const uint32_t* root : roots)
		{
			// the same sentinel in both buffers: the rows neither call writes must match too
			cudaMemset(d_out[0], 0xAB, out_bytes);
			cudaMemset(d_out[1], 0xAB, out_bytes);
			batch.extract_pose_features(d_requests, num_requests, options, offsets, num_offsets, d_bones, 1, bones_per_list, d_parents, d_out[0],
				nullptr, root, nullptr, d_flags);
			if (aclb200_extract_pose_features(device.get(), batch.clipset(), d_requests, num_requests, &options, offsets, num_offsets, d_bones, 1,
				bones_per_list, nullptr, root, d_parents, nullptr, d_out[1], d_flags + 1, nullptr) != ACLB200_OK)
				return 1;
			std::vector<uint8_t> got[2] = { std::vector<uint8_t>(out_bytes), std::vector<uint8_t>(out_bytes) };
			uint32_t flags[2] = { 0, 0 };
			for (int i = 0; i < 2; ++i)
				if (cudaMemcpy(got[i].data(), d_out[i], out_bytes, cudaMemcpyDeviceToHost) != cudaSuccess)
					return 1;
			if (cudaMemcpy(flags, d_flags, sizeof(flags), cudaMemcpyDeviceToHost) != cudaSuccess)
				return 1;
			if (std::memcmp(got[0].data(), got[1].data(), out_bytes) != 0 || flags[0] != flags[1])
			{
				std::printf("FAIL root %s\n", root == nullptr ? "0" : "last");
				return 1;
			}
			// request 7 and every hole stay untouched; request 0's first row is written
			const size_t pose_bytes = size_t(num_offsets) * bones_per_list * 48;
			std::vector<uint8_t> untouched(pose_bytes, 0xAB);
			if (std::memcmp(got[0].data() + 7 * pose_bytes, untouched.data(), pose_bytes) != 0 || std::memcmp(got[0].data() + 2 * 48, untouched.data(), 48) != 0
				|| std::memcmp(got[0].data(), untouched.data(), 48) == 0)
			{
				std::printf("FAIL rows written\n");
				return 1;
			}
		}
		cudaFree(d_requests);
		cudaFree(d_bones);
		cudaFree(d_parents);
		cudaFree(d_roots);
		cudaFree(d_flags);
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
