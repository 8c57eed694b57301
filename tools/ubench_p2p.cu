// Peer-store bandwidth from a kernel (single process, 2 devices) -- context for the exchange numbers.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
typedef uint64_t u64;
__global__ void st8(u64* dst, const u64* src, u64 n){ for (u64 i=(u64)blockIdx.x*blockDim.x+threadIdx.x;i<n;i+=(u64)gridDim.x*blockDim.x) dst[i]=src[i]; }
__global__ void st16(ulonglong2* dst, const ulonglong2* src, u64 n){ for (u64 i=(u64)blockIdx.x*blockDim.x+threadIdx.x;i<n;i+=(u64)gridDim.x*blockDim.x) dst[i]=src[i]; }
int main(){
  int nd=0; cudaGetDeviceCount(&nd); if(nd<2){printf("need 2 GPUs\n");return 0;}
  int can=0; cudaDeviceCanAccessPeer(&can,0,1); printf("canAccessPeer 0->1: %d\n",can);
  u64 n=1ull<<25; u64 *src,*dst_local,*dst_peer;
  cudaSetDevice(1); cudaMalloc(&dst_peer,n*8);
  cudaSetDevice(0); cudaDeviceEnablePeerAccess(1,0); cudaMalloc(&src,n*8); cudaMalloc(&dst_local,n*8); cudaMemset(src,1,n*8);
  cudaEvent_t a,b; cudaEventCreate(&a); cudaEventCreate(&b);
  for (int grid: {132, 132*4, 132*16}){
    for (int mode=0;mode<4;++mode){
      float best=1e9;
      for(int r=0;r<3;++r){ cudaEventRecord(a);
        if(mode==0) st8<<<grid,256>>>(dst_local,src,n); else if(mode==1) st8<<<grid,256>>>(dst_peer,src,n);
        else if(mode==2) st16<<<grid,256>>>((ulonglong2*)dst_peer,(const ulonglong2*)src,n/2); else cudaMemcpyPeerAsync(dst_peer,1,src,0,n*8);
        cudaEventRecord(b); cudaEventSynchronize(b); float ms; cudaEventElapsedTime(&ms,a,b); if(ms<best)best=ms; }
      const char* nm[]={"local st8","peer st8","peer st16","cudaMemcpyPeer"};
      printf("grid %5d %-15s %.3f ms  %.0f GB/s\n",grid,nm[mode],best,n*8/best/1e6);
    }
  }
  printf("err %s\n",cudaGetErrorString(cudaGetLastError()));
}
