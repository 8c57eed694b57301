// Partition kernels alone (all destinations local): is the scatter slow by itself?
#include <cstdio>
#include "../bytewax_b200/csrc/bw_common.cuh"
#include "../bytewax_b200/csrc/bw_exchange.cuh"
__global__ void gen(u64* k, u64* v, u64 n){ for (u64 i=(u64)blockIdx.x*blockDim.x+threadIdx.x;i<n;i+=(u64)gridDim.x*blockDim.x){ k[i]=bw_splitmix64(0x5EEDULL^i)%1000000ULL; v[i]=i; } }
int main(){
  u64 n=1ull<<24; u64 *k,*v; cudaMalloc(&k,n*8); cudaMalloc(&v,n*8); gen<<<1184,256>>>(k,v,n);
  Counters* ctr; cudaMalloc(&ctr,sizeof(Counters)); cudaMemset(ctr,0,sizeof(Counters));
  u32* tc; cudaMalloc(&tc,(n/BW_PART_TILE+1)*BW_MAX_WORLD*4);
  for (int world: {2,4,8}){
    PartIn in{}; in.keys=k; in.vals=v; in.ts=nullptr; in.n=n; in.val_bytes=8; in.world=world;
    PartOut po{}; po.region_cap=n; u64* counts; cudaMalloc(&counts,64);
    for(int d=0;d<world;++d){ cudaMalloc(&po.keys[d],n*8); cudaMalloc(&po.vals[d],n*8); po.counts[d]=counts+d; }
    cudaEvent_t e[4]; for(auto&x:e) cudaEventCreate(&x);
    u64 ntiles=(n+BW_PART_TILE-1)/BW_PART_TILE; int grid=(int)(ntiles<132*8?ntiles:132*8);
    float t[3]={0,0,0};
    for(int rep=0;rep<4;++rep){
      cudaEventRecord(e[0]); k_part_hist<<<grid,BW_PART_THREADS>>>(in,tc);
      cudaEventRecord(e[1]); k_part_scan<<<world,1024>>>(n,world,tc,po,ctr);
      cudaEventRecord(e[2]); k_part_scatter<<<grid,BW_PART_THREADS,(size_t)BW_PART_TILE*16>>>(in,tc,po);
      cudaEventRecord(e[3]); cudaEventSynchronize(e[3]);
      if(rep){ for(int i=0;i<3;++i){ float ms; cudaEventElapsedTime(&ms,e[i],e[i+1]); t[i]+=ms/3; } }
    }
    printf("world %d: hist %.3f ms  scan %.3f ms  scatter %.3f ms  (err %s)\n",world,t[0],t[1],t[2],cudaGetErrorString(cudaGetLastError()));
    for(int d=0;d<world;++d){ cudaFree(po.keys[d]); cudaFree(po.vals[d]); }
  }
}
