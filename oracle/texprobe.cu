// TEST INFRASTRUCTURE ONLY.  Probes what the GPU texture unit returns for the
// input-image texture configuration the reference uses (normalized coordinates,
// bilinear filter, clamp, u8 -> normalized float; /root/reference/src/popsift/s_image.cu:138-167)
// when addressed the way normalizedSource::horiz does (s_pyramid_build_ra.cu:36-53).
// The answers pin the "virtual up-scaled image" formula used by oracle/sift_oracle.c
// and by the product's level-0 kernel.  Our own code; no reference code inside.
//
//   texprobe pairs  out.bin          all 256x256 (a,b) pairs at fraction 0.5 in x, in y,
//                                    and a 2x2 sample; plus fraction 0 for all 256 values
//   texprobe fpairs out.bin         float texture (ImageFloat, s_image.cu:262-291): 2x2 blends of a random
//                                    64x64 float image at a 16x16 grid of fractions, and the fraction quantisation
//   texprobe upairs out.bin         the 8-bit texture at general fractions (16x16 grid, random 64x64 image)
//   texprobe coords W H UP out.bin   random WxH u8 image; for rows 0..7 and the last 8,
//                                    every X in [0,W0) and off in [-16,16]: tex2D at
//                                    ((X+shift)/W0 -/+ off/W0, (Y+shift)/H0); writes image + samples
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include <cmath>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { fprintf(stderr, "CUDA %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); exit(1); } } while (0)

static cudaTextureObject_t make_tex(unsigned char* d, size_t pitch, int w, int h)
{
    cudaTextureDesc td; memset(&td, 0, sizeof(td));
    td.normalizedCoords = 1;
    td.addressMode[0] = td.addressMode[1] = td.addressMode[2] = cudaAddressModeClamp;
    td.readMode = cudaReadModeNormalizedFloat;
    td.filterMode = cudaFilterModeLinear;
    cudaResourceDesc rd; memset(&rd, 0, sizeof(rd));
    rd.resType = cudaResourceTypePitch2D;
    rd.res.pitch2D.devPtr = d;
    rd.res.pitch2D.desc.f = cudaChannelFormatKindUnsigned;
    rd.res.pitch2D.desc.x = 8;
    rd.res.pitch2D.pitchInBytes = pitch;
    rd.res.pitch2D.width = w;
    rd.res.pitch2D.height = h;
    cudaTextureObject_t t; CK(cudaCreateTextureObject(&t, &rd, &td, 0));
    return t;
}

// float texture exactly as ImageFloat::createTexture configures it (s_image.cu:262-291):
// normalized coordinates, bilinear, clamp, cudaReadModeElementType, one 32-bit float channel
static cudaTextureObject_t make_tex_f32(float* d, size_t pitch, int w, int h)
{
    cudaTextureDesc td; memset(&td, 0, sizeof(td));
    td.normalizedCoords = 1;
    td.addressMode[0] = td.addressMode[1] = td.addressMode[2] = cudaAddressModeClamp;
    td.readMode = cudaReadModeElementType;
    td.filterMode = cudaFilterModeLinear;
    cudaResourceDesc rd; memset(&rd, 0, sizeof(rd));
    rd.resType = cudaResourceTypePitch2D;
    rd.res.pitch2D.devPtr = d;
    rd.res.pitch2D.desc.f = cudaChannelFormatKindFloat;
    rd.res.pitch2D.desc.x = 32;
    rd.res.pitch2D.pitchInBytes = pitch;
    rd.res.pitch2D.width = w;
    rd.res.pitch2D.height = h;
    cudaTextureObject_t t; CK(cudaCreateTextureObject(&t, &rd, &td, 0));
    return t;
}

// image: 512 x 256, row a: pixels (2a even cols..)  -> generic fetch kernel
__global__ void fetch(cudaTextureObject_t tex, const float2* xy, float* out, int n)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = tex2D<float>(tex, xy[i].x, xy[i].y);
}

__global__ void coords_kernel(cudaTextureObject_t tex, float* out, int W0, int H0, float shift,
                              const int* rows, int nrows, int maxoff)
{
    int X = blockIdx.x * blockDim.x + threadIdx.x;
    int r = blockIdx.y;
    if (X >= W0) return;
    int Y = rows[r];
    // exactly the reference's coordinate arithmetic
    const float read_x = (blockIdx.x * blockDim.x + threadIdx.x + shift) / W0;
    const float read_y = (Y + shift) / H0;
    int nof = 2 * maxoff + 1;
    float* o = out + (size_t(r) * W0 + X) * nof;
    for (int off = 1; off <= maxoff; off++) {
        const float offrel = float(off) / W0;
        o[maxoff - off] = tex2D<float>(tex, read_x - offrel, read_y);
        o[maxoff + off] = tex2D<float>(tex, read_x + offrel, read_y);
    }
    o[maxoff] = tex2D<float>(tex, read_x, read_y);
}

// unnormalized-coordinate, linear, clamp, layered float texture exactly as Octave::alloc_data_tex / alloc_interm_tex
// configure theirs (sift_octave.cu:243-252,311-325); c = the coordinate handed to tex2DLayered (readTex adds 0.5 itself)
__global__ void lfetch(cudaTextureObject_t tex, const float2* xy, float* out, int n)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = tex2DLayered<float>(tex, xy[i].x, xy[i].y, 0);
}

int main(int argc, char** argv)
{
    if (argc < 3) { fprintf(stderr, "usage\n"); return 2; }
    if (!strcmp(argv[1], "lcoords")) {
        // texprobe lcoords out.bin : texel (x, y) = 256 if (x + y) odd else 0, so a fetch between a zero texel and its
        // right (upper) neighbour returns the 8-bit weight itself.  Sweeps of the x coordinate in steps of 1/4096 around several
        // columns (small and large), the same in y, and the reference's own expression x - off + 0.5 for a few (x, off).
        const int W = 8192, H = 64;
        std::vector<float> img(size_t(W) * H);
        for (int y = 0; y < H; y++) for (int x = 0; x < W; x++) img[size_t(y) * W + x] = ((x + y) & 1) ? 256.0f : 0.0f;
        cudaChannelFormatDesc cd = cudaCreateChannelDesc<float>();
        cudaArray_t arr; CK(cudaMalloc3DArray(&arr, &cd, make_cudaExtent(W, H, 1), cudaArrayLayered));
        cudaMemcpy3DParms cp; memset(&cp, 0, sizeof(cp));
        cp.srcPtr = make_cudaPitchedPtr(img.data(), W * sizeof(float), W, H);
        cp.dstArray = arr; cp.extent = make_cudaExtent(W, H, 1); cp.kind = cudaMemcpyHostToDevice;
        CK(cudaMemcpy3D(&cp));
        cudaResourceDesc rd; memset(&rd, 0, sizeof(rd)); rd.resType = cudaResourceTypeArray; rd.res.array.array = arr;
        cudaTextureDesc td; memset(&td, 0, sizeof(td));
        td.normalizedCoords = 0; td.addressMode[0] = td.addressMode[1] = td.addressMode[2] = cudaAddressModeClamp;
        td.readMode = cudaReadModeElementType; td.filterMode = cudaFilterModeLinear;
        cudaTextureObject_t t; CK(cudaCreateTextureObject(&t, &rd, &td, 0));
        std::vector<float2> q;
        const int cols[] = {0, 1, 2, 5, 64, 1000, 2047, 2048, 4095, 4096, 8000, 8190};
        for (int c : cols) for (int k = -2048; k < 6144; k++) q.push_back(make_float2(float(c) + 0.5f + float(k) / 4096.0f, 10.5f));
        const int rows[] = {0, 1, 2, 31, 62};
        for (int r : rows) for (int k = -2048; k < 6144; k++) q.push_back(make_float2(100.5f, float(r) + 0.5f + float(k) / 4096.0f));
        // the reference's expression: float(x) - off + 0.5f with off = offset + (1 - u), u a float in (0, 1)
        srand(99);
        for (int i = 0; i < 65536; i++) {
            const int x = rand() % 8000 + 40, offset = 1 + 2 * (rand() % 8);
            const float u = float(rand() % 1000000) / 1000000.0f;
            const float off = offset + (1.0f - u);
            q.push_back(make_float2((float(x) - off) + 0.5f, 20.5f));
            q.push_back(make_float2((float(x) + off) + 0.5f, 20.5f));
        }
        float2* dq; float* dout; CK(cudaMalloc(&dq, q.size() * sizeof(float2))); CK(cudaMalloc(&dout, q.size() * 4));
        CK(cudaMemcpy(dq, q.data(), q.size() * sizeof(float2), cudaMemcpyHostToDevice));
        lfetch<<<(int(q.size()) + 255) / 256, 256>>>(t, dq, dout, int(q.size()));
        CK(cudaDeviceSynchronize());
        std::vector<float> o(q.size()); CK(cudaMemcpy(o.data(), dout, q.size() * 4, cudaMemcpyDeviceToHost));
        FILE* fp = fopen(argv[2], "wb");
        int hdr[4] = { W, H, int(q.size()), 0 };
        fwrite(hdr, 4, 4, fp); fwrite(q.data(), sizeof(float2), q.size(), fp); fwrite(o.data(), 4, o.size(), fp);
        fclose(fp);
        printf("texprobe lcoords: %zu samples\n", q.size());
        return 0;
    }
    if (!strcmp(argv[1], "pairs")) {
        // image 512 wide x 512 high:
        //   rows 0..255   : row a holds [a, b] pairs at columns (2b, 2b+1)  -> x-fraction 0.5 between them
        //   we build separate images for x and y tests to keep it simple.
        const int W = 512, H = 256;
        std::vector<unsigned char> img(size_t(W) * H);
        for (int a = 0; a < 256; a++) for (int b = 0; b < 256; b++) { img[size_t(a) * W + 2 * b] = a; img[size_t(a) * W + 2 * b + 1] = b; }
        unsigned char* d; size_t pitch; CK(cudaMallocPitch(&d, &pitch, W, H));
        CK(cudaMemcpy2D(d, pitch, img.data(), W, W, H, cudaMemcpyHostToDevice));
        cudaTextureObject_t tx = make_tex(d, pitch, W, H);
        // x pairs: sample between col 2b and 2b+1 of row a: texel coord u = 2b+0.5(+0.5 centre) -> normalized (2b+1)/W
        std::vector<float2> xy; xy.reserve(65536 * 2 + 256);
        for (int a = 0; a < 256; a++) for (int b = 0; b < 256; b++) xy.push_back(make_float2((2 * b + 1.0f) / W, (a + 0.5f) / H));
        // fraction 0: centre of texel (2b) in row 0..: value b' = img[0][2b]=0 ... use row a col 0 -> value a
        for (int a = 0; a < 256; a++) xy.push_back(make_float2(0.5f / W, (a + 0.5f) / H));
        // y pairs: image2 W2=256,H2=512: col a, rows (2b,2b+1)
        const int W2 = 256, H2 = 512;
        std::vector<unsigned char> img2(size_t(W2) * H2);
        for (int a = 0; a < 256; a++) for (int b = 0; b < 256; b++) { img2[size_t(2 * b) * W2 + a] = a; img2[size_t(2 * b + 1) * W2 + a] = b; }
        unsigned char* d2; size_t pitch2; CK(cudaMallocPitch(&d2, &pitch2, W2, H2));
        CK(cudaMemcpy2D(d2, pitch2, img2.data(), W2, W2, H2, cudaMemcpyHostToDevice));
        cudaTextureObject_t ty = make_tex(d2, pitch2, W2, H2);
        std::vector<float2> xy2;
        for (int a = 0; a < 256; a++) for (int b = 0; b < 256; b++) xy2.push_back(make_float2((a + 0.5f) / W2, (2 * b + 1.0f) / H2));
        // 2x2: random image 64x64, sample at every corner point (x+1)/W,(y+1)/H for x,y<63
        const int W3 = 64, H3 = 64;
        std::vector<unsigned char> img3(W3 * H3); srand(7); for (auto& v : img3) v = rand() & 255;
        unsigned char* d3; size_t pitch3; CK(cudaMallocPitch(&d3, &pitch3, W3, H3));
        CK(cudaMemcpy2D(d3, pitch3, img3.data(), W3, W3, H3, cudaMemcpyHostToDevice));
        cudaTextureObject_t t4 = make_tex(d3, pitch3, W3, H3);
        std::vector<float2> xy3;
        for (int y = 0; y < 63; y++) for (int x = 0; x < 63; x++) xy3.push_back(make_float2((x + 1.0f) / W3, (y + 1.0f) / H3));

        FILE* fp = fopen(argv[2], "wb");
        auto run = [&](cudaTextureObject_t t, std::vector<float2>& q) {
            float2* dq; float* dout; CK(cudaMalloc(&dq, q.size() * sizeof(float2))); CK(cudaMalloc(&dout, q.size() * 4));
            CK(cudaMemcpy(dq, q.data(), q.size() * sizeof(float2), cudaMemcpyHostToDevice));
            fetch<<<(int(q.size()) + 255) / 256, 256>>>(t, dq, dout, int(q.size()));
            CK(cudaDeviceSynchronize());
            std::vector<float> o(q.size()); CK(cudaMemcpy(o.data(), dout, q.size() * 4, cudaMemcpyDeviceToHost));
            int n = int(q.size()); fwrite(&n, 4, 1, fp); fwrite(o.data(), 4, n, fp);
            cudaFree(dq); cudaFree(dout);
        };
        run(tx, xy); run(ty, xy2);
        fwrite(img3.data(), 1, img3.size(), fp);
        run(t4, xy3);
        fclose(fp);
        printf("texprobe pairs: done\n");
        return 0;
    }
    if (!strcmp(argv[1], "fpairs")) {
        // 64x64 float image (power-of-two size: normalized -> texel coordinates are exact).  Left half of
        // the values are k/256 (what popsift-demo --float-mode feeds, main.cpp:234), right half random
        // 24-bit floats in [0,1).  Samples: for texel (i,j) in [8,40)x[8,40) and fractions (a,b)/256 with
        // a,b in {0,17,...,255}: tex2D at ((i+0.5+a/256)/64, (j+0.5+b/256)/64); then the same texels at the
        // finer fractions a/1024 (b = 0) to see how the fraction is quantised.
        const int W = 64, H = 64;
        std::vector<float> img(size_t(W) * H);
        srand(12345);
        for (int y = 0; y < H; y++) for (int x = 0; x < W; x++)
            img[size_t(y) * W + x] = x < W / 2 ? float(rand() & 255) / 256.0f : float(rand() & 0xffffff) / 16777216.0f;
        float* d; size_t pitch; CK(cudaMallocPitch((void**)&d, &pitch, W * sizeof(float), H));
        CK(cudaMemcpy2D(d, pitch, img.data(), W * sizeof(float), W * sizeof(float), H, cudaMemcpyHostToDevice));
        cudaTextureObject_t t = make_tex_f32(d, pitch, W, H);
        std::vector<float2> q;
        for (int j = 8; j < 40; j++) for (int i = 8; i < 40; i++)
            for (int b = 0; b < 256; b += 17) for (int a = 0; a < 256; a += 17)
                q.push_back(make_float2((i + 0.5f + a / 256.0f) / W, (j + 0.5f + b / 256.0f) / H));
        const int n1 = int(q.size());
        for (int j = 8; j < 12; j++) for (int i = 8; i < 40; i++)
            for (int a = 0; a < 1024; a++) q.push_back(make_float2((i + 0.5f + a / 1024.0f) / W, (j + 0.5f) / H));
        const int n2 = int(q.size()) - n1;
        float2* dq; float* dout; CK(cudaMalloc(&dq, q.size() * sizeof(float2))); CK(cudaMalloc(&dout, q.size() * 4));
        CK(cudaMemcpy(dq, q.data(), q.size() * sizeof(float2), cudaMemcpyHostToDevice));
        fetch<<<(int(q.size()) + 255) / 256, 256>>>(t, dq, dout, int(q.size()));
        CK(cudaDeviceSynchronize());
        std::vector<float> o(q.size()); CK(cudaMemcpy(o.data(), dout, q.size() * 4, cudaMemcpyDeviceToHost));
        FILE* fp = fopen(argv[2], "wb");
        int hdr[4] = { W, H, n1, n2 };
        fwrite(hdr, 4, 4, fp); fwrite(img.data(), 4, img.size(), fp); fwrite(o.data(), 4, o.size(), fp);
        fclose(fp);
        printf("texprobe fpairs: %d + %d samples\n", n1, n2);
        return 0;
    }
    if (!strcmp(argv[1], "upairs")) {
        // the 8-bit texture at GENERAL fractions (the reference's configuration, s_image.cu:138-167): same
        // sampling pattern as fpairs on a random 64x64 u8 image
        const int W = 64, H = 64;
        std::vector<unsigned char> img(size_t(W) * H);
        srand(4321);
        for (auto& v : img) v = rand() & 255;
        unsigned char* d; size_t pitch; CK(cudaMallocPitch((void**)&d, &pitch, W, H));
        CK(cudaMemcpy2D(d, pitch, img.data(), W, W, H, cudaMemcpyHostToDevice));
        cudaTextureObject_t t = make_tex(d, pitch, W, H);
        std::vector<float2> q;
        for (int j = 8; j < 40; j++) for (int i = 8; i < 40; i++)
            for (int b = 0; b < 256; b += 17) for (int a = 0; a < 256; a += 17)
                q.push_back(make_float2((i + 0.5f + a / 256.0f) / W, (j + 0.5f + b / 256.0f) / H));
        const int n1 = int(q.size());
        float2* dq; float* dout; CK(cudaMalloc(&dq, q.size() * sizeof(float2))); CK(cudaMalloc(&dout, q.size() * 4));
        CK(cudaMemcpy(dq, q.data(), q.size() * sizeof(float2), cudaMemcpyHostToDevice));
        fetch<<<(int(q.size()) + 255) / 256, 256>>>(t, dq, dout, int(q.size()));
        CK(cudaDeviceSynchronize());
        std::vector<float> o(q.size()); CK(cudaMemcpy(o.data(), dout, q.size() * 4, cudaMemcpyDeviceToHost));
        FILE* fp = fopen(argv[2], "wb");
        int hdr[4] = { W, H, n1, 0 };
        fwrite(hdr, 4, 4, fp); fwrite(img.data(), 1, img.size(), fp); fwrite(o.data(), 4, o.size(), fp);
        fclose(fp);
        printf("texprobe upairs: %d samples\n", n1);
        return 0;
    }
    if (!strcmp(argv[1], "coords")) {
        int w = atoi(argv[2]), h = atoi(argv[3]); float up = atof(argv[4]); const char* out = argv[5];
        int W0 = (int)ceilf(w * powf(2.0f, up)), H0 = (int)ceilf(h * powf(2.0f, up));
        float shift = 0.5f * powf(2.0f, up);
        std::vector<unsigned char> img(size_t(w) * h); srand(w * 31 + h); for (auto& v : img) v = rand() & 255;
        unsigned char* d; size_t pitch; CK(cudaMallocPitch(&d, &pitch, w, h));
        CK(cudaMemcpy2D(d, pitch, img.data(), w, w, h, cudaMemcpyHostToDevice));
        cudaTextureObject_t t = make_tex(d, pitch, w, h);
        const int maxoff = 16;
        std::vector<int> rows; for (int i = 0; i < 8; i++) rows.push_back(i); for (int i = 8; i >= 1; i--) rows.push_back(H0 - i);
        rows.push_back(H0 / 2); rows.push_back(H0 / 2 + 1);
        int nrows = int(rows.size());
        int* drows; CK(cudaMalloc(&drows, nrows * 4)); CK(cudaMemcpy(drows, rows.data(), nrows * 4, cudaMemcpyHostToDevice));
        size_t n = size_t(nrows) * W0 * (2 * maxoff + 1);
        float* dout; CK(cudaMalloc(&dout, n * 4));
        dim3 grid((W0 + 127) / 128, nrows);
        coords_kernel<<<grid, 128>>>(t, dout, W0, H0, shift, drows, nrows, maxoff);
        CK(cudaDeviceSynchronize());
        std::vector<float> o(n); CK(cudaMemcpy(o.data(), dout, n * 4, cudaMemcpyDeviceToHost));
        FILE* fp = fopen(out, "wb");
        int hdr[6] = { w, h, W0, H0, nrows, maxoff };
        fwrite(hdr, 4, 6, fp); fwrite(rows.data(), 4, nrows, fp);
        fwrite(img.data(), 1, img.size(), fp); fwrite(o.data(), 4, n, fp);
        fclose(fp);
        printf("texprobe coords %dx%d up=%g: done\n", w, h, up);
        return 0;
    }
    return 2;
}
