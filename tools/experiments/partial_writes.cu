// Development experiment: what do partial-sector global stores of 40 byte bones cost in DRAM traffic on an H100?
// mode 0: each thread writes only the 16 byte rotation of its bone (28 of 40 bytes untouched)
// mode 1: each thread writes rotation (16 B), translation (12 B), scale (12 B) of its bone back to back
// mode 2: like 1, but translation+scale are written by a different warp of the block, one "chunk" later
// mode 3: like 1, but rows were first filled by a bulk memcpy-like pass of the same block (base pose) 8 rows earlier
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
__global__ void k(uint8_t* out, uint64_t bones, int mode)
{
	const uint64_t stride = uint64_t(gridDim.x) * blockDim.x;
	for (uint64_t b = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; b < bones; b += stride)
	{
		uint8_t* bone = out + b * 40;
		const float v = float(b);
		if (mode != 2 || (threadIdx.x >> 5) % 2 == 0)
		{
			*reinterpret_cast<float2*>(bone) = make_float2(v, v);
			*reinterpret_cast<float2*>(bone + 8) = make_float2(v, v);
		}
		if (mode == 1)
		{
			*reinterpret_cast<float2*>(bone + 16) = make_float2(v, v);
			*reinterpret_cast<float*>(bone + 24) = v;
			*reinterpret_cast<float*>(bone + 28) = v;
			*reinterpret_cast<float2*>(bone + 32) = make_float2(v, v);
		}
		if (mode == 2)
		{
			// the odd warps write the vectors of the bones the even warp next to them wrote the rotations of, and vice versa
			const uint64_t partner = b ^ 32;
			uint8_t* other = out + partner * 40;
			if ((threadIdx.x >> 5) % 2 == 1)
			{
				*reinterpret_cast<float2*>(bone) = make_float2(v, v);
				*reinterpret_cast<float2*>(bone + 8) = make_float2(v, v);
			}
			__syncthreads();
			if (partner < bones)
			{
				*reinterpret_cast<float2*>(other + 16) = make_float2(v, v);
				*reinterpret_cast<float*>(other + 24) = v;
				*reinterpret_cast<float*>(other + 28) = v;
				*reinterpret_cast<float2*>(other + 32) = make_float2(v, v);
			}
		}
	}
}
int main()
{
	const uint64_t bones = 60000000ull;
	uint8_t* out;
	cudaMalloc(&out, bones * 40);
	cudaMemset(out, 0, bones * 40);
	for (int mode = 0; mode < 3; ++mode)
	{
		cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
		k<<<132 * 8, 256>>>(out, bones, mode);
		cudaEventRecord(a);
		k<<<132 * 8, 256>>>(out, bones, mode);
		cudaEventRecord(b); cudaEventSynchronize(b);
		float ms; cudaEventElapsedTime(&ms, a, b);
		printf("mode %d: %.3f ms (%.1f GB/s of 2.4 GB)\n", mode, ms, 2.4 / ms * 1000);
	}
	return 0;
}
