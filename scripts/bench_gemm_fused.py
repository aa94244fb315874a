"""Attribute the cost of hrl_gemm_fused's operand transforms / epilogues at the tower shape (M x 288 x 288)."""
import ctypes as C, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from handyrl_b200 import nets, tower
from handyrl_b200._capi import lib

M = 16384
eng = tower.FusedBoardNet(nets.tictactoe_net().cuda(), M, torch.device('cuda'))
D = eng.D
X = torch.randn(M, D, device='cuda'); Y = torch.randn(M, D, device='cuda'); W = torch.randn(D, D, device='cuda') * 0.1
out = torch.empty(M, D, device='cuda')
c = [torch.rand(D, device='cuda') for _ in range(5)]

def timeit(fn, reps=20):
    """20 launches captured in a CUDA graph (no host launch overhead between them), replayed 5 times."""
    for _ in range(3): fn()
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            for _ in range(reps): fn()
        graph.replay(); side.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(side)
        for _ in range(5): graph.replay()
        e1.record(side); side.synchronize()
    return e0.elapsed_time(e1) / (5 * reps) * 1e3

Wf, Wb = eng.Wf[0], eng.Wb[0]      # packed images (contents irrelevant for timing)
ep_full = dict(y=Y, scale=c[0], shift=c[1], mean=c[2], rstd=c[3])
cases = {
    'fwd plain': lambda: eng._gemm(dict(t=X), dict(t=W), out, K=D, N=D),
    'fwd relu epilogue': lambda: eng._gemm(dict(t=X), dict(t=W), out, K=D, N=D, epilogue='relu'),
    'fwd stats epilogue': lambda: eng._gemm(dict(t=X), dict(t=W), out, K=D, N=D, epilogue='stats'),
    'fwd A affine+relu': lambda: eng._gemm(dict(t=X, consts=(c[0], c[1]), relu=True), dict(t=W), out, K=D, N=D),
    'fwd A affine+relu + stats': lambda: eng._gemm(dict(t=X, consts=(c[0], c[1]), relu=True), dict(t=W), out, K=D, N=D, epilogue='stats'),
    'fwd packed B': lambda: eng._gemm(dict(t=X), dict(t=Wf, packed=True), out, K=D, N=D),
    'fwd packed B, A affine+relu + stats': lambda: eng._gemm(dict(t=X, consts=(c[0], c[1]), relu=True), dict(t=Wf, packed=True), out, K=D, N=D,
                                                              epilogue='stats'),
    'dgrad packed B, 2-source + mask_stats': lambda: eng._gemm(dict(t=X, t2=Y, consts=(c[0], c[1], c[2])), dict(t=Wb, packed=True), out, K=D,
                                                                N=D, epilogue='mask_stats', ep=ep_full),
    'dgrad plain': lambda: eng._gemm(dict(t=X), dict(t=W, kmajor=False), out, K=D, N=D),
    'dgrad A 2-source': lambda: eng._gemm(dict(t=X, t2=Y, consts=(c[0], c[1], c[2])), dict(t=W, kmajor=False), out, K=D, N=D),
    'dgrad A 2-source + mask_stats': lambda: eng._gemm(dict(t=X, t2=Y, consts=(c[0], c[1], c[2])), dict(t=W, kmajor=False), out, K=D, N=D,
                                                       epilogue='mask_stats', ep=ep_full),
    'dgrad plain + mask_stats': lambda: eng._gemm(dict(t=X), dict(t=W, kmajor=False), out, K=D, N=D, epilogue='mask_stats', ep=ep_full),
    'wgrad plain (48 slices, partials)': lambda: eng._gemm(dict(t=X, kmajor=False), dict(t=Y, kmajor=False), None, K=M, N=D, M=D, splits=eng.splits['tower'], partial=True, ws=eng.ws),
    'wgrad both transformed': lambda: eng._gemm(dict(t=X, t2=Y, consts=(c[0], c[1], c[2]), kmajor=False, by_row=True),
                                                dict(t=Y, consts=(c[3], c[4]), relu=True, kmajor=False, by_row=True), None, K=M, N=D, M=D,
                                                splits=eng.splits['tower'], partial=True, ws=eng.ws),
}
for k, fn in (cases.items() if __name__ == "__main__" else ()):
    print('%-40s %6.1f us' % (k, timeit(fn)))
g = torch.empty(32, 32, 3, 3, device='cuda')
print('%-36s %6.1f us' % ('fold (48 slices)', timeit(lambda: lib().hrl_board_fold(eng.ws.data_ptr(), eng.splits['tower'], D * D, g.data_ptr(), 32, 32, 3, 3, 3, 3, torch.cuda.current_stream().cuda_stream))))
