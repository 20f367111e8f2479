// tests/cpp/shim_additive.cpp -- acl_b200::batch_decompressor::decompress_tracks_additive and apply_additive_to_base against the C calls
// they wrap: the clip layered on itself at other sample times, every format, local rows and object space rows (a binary tree), then the
// standalone call on the local rows; the outputs must be byte-identical.
// usage: shim_additive <clip.acl.bin>; prints PASS, exits 3 without a CUDA device.
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
		std::vector<aclb200_additive_request> requests;
		for (uint32_t i = 0; i < 64; ++i)
			requests.push_back(aclb200_additive_request{ aclb200_request{ 0u, float(i) * 0.037f - 0.1f }, aclb200_request{ 0u, float(63 - i) * 0.029f } });
		std::vector<uint32_t> parents(num_tracks);
		for (uint32_t bone = 0; bone < num_tracks; ++bone)
			parents[bone] = bone == 0 ? 0xFFFFFFFFu : (bone - 1) / 2;
		const size_t out_bytes = size_t(num_tracks) * 48 * requests.size();
		aclb200_additive_request* d_requests = nullptr;
		uint32_t* d_parents = nullptr;
		uint8_t* d_out[2] = { nullptr, nullptr };
		if (cudaMalloc(&d_requests, requests.size() * sizeof(aclb200_additive_request)) != cudaSuccess || cudaMalloc(&d_parents, num_tracks * sizeof(uint32_t)) != cudaSuccess
			|| cudaMalloc(&d_out[0], out_bytes) != cudaSuccess || cudaMalloc(&d_out[1], out_bytes) != cudaSuccess)
			return 1;
		cudaMemcpy(d_requests, requests.data(), requests.size() * sizeof(aclb200_additive_request), cudaMemcpyHostToDevice);
		cudaMemcpy(d_parents, parents.data(), num_tracks * sizeof(uint32_t), cudaMemcpyHostToDevice);
		aclb200_options options;
		aclb200_default_options(&options);
		const uint32_t num_requests = uint32_t(requests.size());
		const auto same = [&](const char* what, uint32_t format) -> bool
		{
			std::vector<uint8_t> got[2] = { std::vector<uint8_t>(out_bytes), std::vector<uint8_t>(out_bytes) };
			for (int i = 0; i < 2; ++i)
				if (cudaMemcpy(got[i].data(), d_out[i], out_bytes, cudaMemcpyDeviceToHost) != cudaSuccess)
					return false;
			if (std::memcmp(got[0].data(), got[1].data(), out_bytes) == 0)
				return true;
			std::printf("FAIL %s format %u\n", what, format);
			return false;
		};
		for (uint32_t format = ACLB200_ADDITIVE_NONE; format <= ACLB200_ADDITIVE_ADDITIVE1; ++format)
		{
			for (const uint32_t* parent_pointer : { static_cast<const uint32_t*>(nullptr), static_cast<const uint32_t*>(d_parents) })
			{
				cudaMemset(d_out[0], 0xAB, out_bytes);
				cudaMemset(d_out[1], 0xCD, out_bytes);
				batch.decompress_tracks_additive(d_requests, num_requests, options, format, nullptr, d_out[0], parent_pointer);
				if (aclb200_decompress_tracks_additive(device.get(), batch.clipset(), d_requests, num_requests, &options, format, nullptr, parent_pointer, nullptr,
					ACLB200_OBJECT_QVVF, d_out[1], nullptr, nullptr) != ACLB200_OK)
					return 1;
				if (!same(parent_pointer != nullptr ? "object space" : "local", format))
					return 1;
			}
			// the standalone call over the local rows: in place through the shim, into the other buffer through the C call
			batch.decompress_tracks_additive(d_requests, num_requests, options, format, nullptr, d_out[0]);
			cudaMemcpy(d_out[1], d_out[0], out_bytes, cudaMemcpyDeviceToDevice);
			batch.apply_additive_to_base(d_out[0], d_out[0], d_out[0], num_requests, num_tracks, format);
			if (aclb200_apply_additive_to_base(device.get(), d_out[1], d_out[1], d_out[1], num_requests, num_tracks, 0, format, nullptr, nullptr) != ACLB200_OK)
				return 1;
			if (!same("apply_additive_to_base", format))
				return 1;
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
