// tests/cpp/shim_object_space.cpp -- acl_b200::batch_decompressor::decompress_tracks_object_space against the C call it wraps: one
// launch through each, same clip, requests, options and skeleton (a binary tree), both object kinds; the outputs must be byte-identical.
// usage: shim_object_space <clip.acl.bin>; prints PASS, exits 3 without a CUDA device.
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
		std::vector<aclb200_request> requests;
		for (uint32_t i = 0; i < 64; ++i)
			requests.push_back(aclb200_request{ 0u, float(i) * 0.037f - 0.1f });
		std::vector<uint32_t> parents(num_tracks);
		for (uint32_t bone = 0; bone < num_tracks; ++bone)
			parents[bone] = bone == 0 ? 0xFFFFFFFFu : (bone - 1) / 2;
		const size_t pose_bytes = size_t(num_tracks) * 48, out_bytes = pose_bytes * requests.size();
		aclb200_request* d_requests = nullptr;
		uint32_t* d_parents = nullptr;
		uint8_t* d_out[2] = { nullptr, nullptr };
		if (cudaMalloc(&d_requests, requests.size() * sizeof(aclb200_request)) != cudaSuccess || cudaMalloc(&d_parents, num_tracks * sizeof(uint32_t)) != cudaSuccess
			|| cudaMalloc(&d_out[0], out_bytes) != cudaSuccess || cudaMalloc(&d_out[1], out_bytes) != cudaSuccess)
			return 1;
		cudaMemcpy(d_requests, requests.data(), requests.size() * sizeof(aclb200_request), cudaMemcpyHostToDevice);
		cudaMemcpy(d_parents, parents.data(), num_tracks * sizeof(uint32_t), cudaMemcpyHostToDevice);
		aclb200_options options;
		aclb200_default_options(&options);
		for (uint32_t kind : { uint32_t(ACLB200_OBJECT_QVVF), uint32_t(ACLB200_OBJECT_MATRIX3X4F) })
		{
			cudaMemset(d_out[0], 0xAB, out_bytes);
			cudaMemset(d_out[1], 0xCD, out_bytes);
			batch.decompress_tracks_object_space(d_requests, uint32_t(requests.size()), options, d_parents, nullptr, kind, d_out[0]);
			if (aclb200_decompress_tracks_object_space(device.get(), batch.clipset(), d_requests, uint32_t(requests.size()), &options, d_parents, nullptr, kind,
				d_out[1], nullptr, nullptr) != ACLB200_OK)
				return 1;
			std::vector<uint8_t> got[2] = { std::vector<uint8_t>(out_bytes), std::vector<uint8_t>(out_bytes) };
			for (int i = 0; i < 2; ++i)
				if (cudaMemcpy(got[i].data(), d_out[i], out_bytes, cudaMemcpyDeviceToHost) != cudaSuccess)
					return 1;
			if (std::memcmp(got[0].data(), got[1].data(), out_bytes) != 0)
			{
				std::printf("FAIL kind %u\n", kind);
				return 1;
			}
		}
		cudaFree(d_requests);
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
